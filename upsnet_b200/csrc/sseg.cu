// sseg.cu -- semantic-segmentation confusion matrix of one image (evaluation half of SURVEY section 8f row f4), device
// resident:
//
//  * upsnet_sseg_update: dataset/cityscapes.py:445-467 / coco.py:225-247 evaluate_ssegs for one image -- the prediction
//    written as np.uint8 (values wrap mod 256), resized to the ground truth with Pillow's NEAREST rule, pixels with
//    gt == 255 dropped -- composed with base_dataset.py:806-824 get_confusion_matrix (bin gt * C + pred, bins >= C*C
//    dropped).  Reference: a PNG round trip, PIL resize and np.bincount on the host.
//    Here: one pass over the ground-truth pixels that gathers the prediction through two index tables (all resize and
//    restore geometry is in the tables, built on the host), counts into a per-block shared-memory histogram of C*C bins
//    with warp-aggregated adds, and flushes the non-zero bins to the int64 accumulator with integer atomics (the
//    result does not depend on the order of the adds).  HBM-bound: 1 byte of gt plus one prediction element per pixel.
#include "common.cuh"

namespace ups {

constexpr int kSsegThreads = 256;
constexpr int kSsegMaxClasses = UPSNET_SSEG_MAX_CLASSES;
constexpr unsigned kSsegNone = 0xffffffffu;

// 4 consecutive gt pixels per thread per step (one 32-bit gt load when aligned).  Equal bins of a thread's 4 pixels merge
// into runs; the lanes of a warp holding the same run bin elect one leader that adds the run lengths (as pq_pixel_kernel).
template <typename T>
__global__ void __launch_bounds__(kSsegThreads)
sseg_kernel(const T* __restrict__ pred, int pitch, const int* __restrict__ row_src, const int* __restrict__ col_src,
            const unsigned char* __restrict__ gt, int W, size_t HW, int C, unsigned long long* __restrict__ acc) {
  extern __shared__ unsigned sseg_hist[];
  const unsigned CC = (unsigned)C * (unsigned)C;
  for (unsigned t = threadIdx.x; t < CC; t += blockDim.x) sseg_hist[t] = 0u;
  __syncthreads();
  const bool vec = (reinterpret_cast<uintptr_t>(gt) & 3) == 0;
  const size_t nq = (HW + 3) / 4;
  for (size_t q0 = (size_t)blockIdx.x * blockDim.x; q0 < nq; q0 += (size_t)gridDim.x * blockDim.x) {
    const size_t q = q0 + threadIdx.x;
    unsigned key[4] = {kSsegNone, kSsegNone, kSsegNone, kSsegNone};
    if (q < nq) {
      unsigned g4 = 0u;
      int np = 4;
      if (vec && 4 * q + 4 <= HW) {
        g4 = __ldg(reinterpret_cast<const unsigned*>(gt) + q);
      } else {
        np = (int)min((size_t)4, HW - 4 * q);
        for (int b = 0; b < np; ++b) g4 |= (unsigned)gt[4 * q + b] << (8 * b);
      }
      int y = (int)(4 * q / W), x = (int)(4 * q - (size_t)y * W);
      const T* prow = pred + (size_t)__ldg(row_src + y) * pitch;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (j >= np) break;
        const unsigned g = (g4 >> (8 * j)) & 0xffu;
        if (g != 255u) {                                        // ignore label: the prediction is not read
          const unsigned p = (unsigned)(unsigned char)prow[__ldg(col_src + x)];     // np.uint8: wraps mod 256
          const unsigned f = g * (unsigned)C + p;
          if (f < CC) key[j] = f;                               // gt >= C rows and aliases past the last bin drop
        }
        if (++x == W && j + 1 < np) {
          x = 0;
          prow = pred + (size_t)__ldg(row_src + ++y) * pitch;
        }
      }
    }
    // runs of equal bins: the run starting at pixel j has bin rk[j] and length rc[j] (static indices: no local memory)
    unsigned rk[4], rc[4];
    rc[3] = 1u;
#pragma unroll
    for (int j = 2; j >= 0; --j) rc[j] = key[j + 1] == key[j] ? rc[j + 1] + 1u : 1u;
#pragma unroll
    for (int j = 0; j < 4; ++j) rk[j] = (j == 0 || key[j - 1] != key[j]) ? key[j] : kSsegNone;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (!__any_sync(0xffffffffu, rk[j] != kSsegNone)) continue;
      const unsigned peers = __match_any_sync(0xffffffffu, rk[j]);
      const unsigned sum = __reduce_add_sync(peers, rc[j]);
      if (rk[j] != kSsegNone && (int)(__ffs(peers) - 1) == (int)(threadIdx.x & 31)) atomicAdd(sseg_hist + rk[j], sum);
    }
  }
  __syncthreads();
  for (unsigned t = threadIdx.x; t < CC; t += blockDim.x) {
    const unsigned c = sseg_hist[t];
    if (c) atomicAdd(acc + t, (unsigned long long)c);
  }
}

template <typename T>
static int sseg_launch(const void* pred, int pitch, const int* row_src, const int* col_src, const unsigned char* gt, int H,
                       int W, int C, long long* acc, cudaStream_t st) {
  static PerDeviceOnce configured;
  if (configured.need())
    UPS_CUDA(cudaFuncSetAttribute(sseg_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)(sizeof(unsigned) * kSsegMaxClasses * kSsegMaxClasses)));
  const size_t smem = sizeof(unsigned) * (size_t)C * C;
  int per_sm = 0;
  UPS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, sseg_kernel<T>, kSsegThreads, smem));
  const size_t HW = (size_t)H * W, nq = (HW + 3) / 4;
  size_t blocks = (nq + kSsegThreads - 1) / kSsegThreads;             // persistent: each block zeroes and flushes C*C bins
  if (blocks > (size_t)num_sms() * max(per_sm, 1)) blocks = (size_t)num_sms() * max(per_sm, 1);
  sseg_kernel<T><<<(unsigned)blocks, kSsegThreads, smem, st>>>((const T*)pred, pitch, row_src, col_src, gt, W, HW, C,
                                                                 reinterpret_cast<unsigned long long*>(acc));
  UPS_CHECK_LAUNCH();
  return 0;
}

}  // namespace ups

extern "C" int upsnet_sseg_update(const void* pred, int pred_bytes, int pred_pitch, const int* row_src, const int* col_src,
                                  const unsigned char* gt, int H, int W, int num_classes, long long* acc, void* stream) {
  using namespace ups;
  if (!pred || !row_src || !col_src || !gt || !acc) return UPSNET_E_BADARG;
  if (H <= 0 || W <= 0 || pred_pitch <= 0 || num_classes < 1 || num_classes > kSsegMaxClasses) return UPSNET_E_BADARG;
  cudaStream_t st = (cudaStream_t)stream;
  if (pred_bytes == 1) return sseg_launch<unsigned char>(pred, pred_pitch, row_src, col_src, gt, H, W, num_classes, acc, st);
  if (pred_bytes == 8) return sseg_launch<long long>(pred, pred_pitch, row_src, col_src, gt, H, W, num_classes, acc, st);
  return UPSNET_E_BADARG;
}
