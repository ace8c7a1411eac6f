// nms.cu -- device-resident, segmented greedy NMS for sm_90a.
//
// Semantics: nms/nms_kernel.cu:30-38 (devIoU with +1 areas), :77 (suppress IoU > thresh) and
// the greedy sweep of :130-146 -- which the reference runs on the HOST after a D2H copy of the
// bitmask -- here performed on the device, so nothing crosses PCIe and S independent problems
// (5 RPN levels, or the per-class problems of MaskROI) share one launch pair.
//
// Kernel 1 (nms_mask_kernel): 64x64-tile IoU bitmask, upper-triangular tiles only (the sweep
//   never reads tiles with col < row, nms_kernel.cu:139).
// Kernel 2 (nms_sweep_kernel): one CTA per segment walks 64-box blocks: a single thread
//   resolves the 64x64 diagonal word serially (64 dependent steps on registers), then all
//   threads OR the kept rows into the running `removed` words held in shared memory.
// Latency-bound for N~1000 (148 KB of algorithmic bytes); reported as us/call (DESIGN.md).
#include "common.cuh"

namespace ups {

constexpr int kNmsTile = 64;
constexpr int kNmsMaxSeg = 65536;

__device__ __forceinline__ float dev_iou(const float4 a, const float4 b) {
  // explicit _rn intrinsics: no FMA contraction, so the `> thresh` decision is bit-identical
  // to the un-fused fp32 arithmetic of py_cpu_nms.py / the C oracle.
  const float left = fmaxf(a.x, b.x), right = fminf(a.z, b.z);
  const float top = fmaxf(a.y, b.y), bottom = fminf(a.w, b.w);
  const float width = fmaxf(__fadd_rn(__fsub_rn(right, left), 1.f), 0.f);
  const float height = fmaxf(__fadd_rn(__fsub_rn(bottom, top), 1.f), 0.f);
  const float interS = __fmul_rn(width, height);
  const float Sa = __fmul_rn(__fadd_rn(__fsub_rn(a.z, a.x), 1.f), __fadd_rn(__fsub_rn(a.w, a.y), 1.f));
  const float Sb = __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), 1.f), __fadd_rn(__fsub_rn(b.w, b.y), 1.f));
  return __fdiv_rn(interS, __fsub_rn(__fadd_rn(Sa, Sb), interS));
}

// grid (col_tiles, row_tiles, S), block 64
__global__ void __launch_bounds__(kNmsTile)
nms_mask_kernel(const float* __restrict__ boxes, const int* __restrict__ seg_offsets,
                int max_seg_len, float thresh, unsigned long long* __restrict__ mask) {
  const int seg = blockIdx.z;
  const int row_t = blockIdx.y, col_t = blockIdx.x;
  if (col_t < row_t) return;
  const int beg = seg_offsets[seg];
  const int n = min(seg_offsets[seg + 1] - beg, max_seg_len);
  if (row_t * kNmsTile >= n || col_t * kNmsTile >= n) return;
  const int row_size = min(n - row_t * kNmsTile, kNmsTile);
  const int col_size = min(n - col_t * kNmsTile, kNmsTile);
  const int max_cb = ceil_div(max_seg_len, kNmsTile);
  unsigned long long* seg_mask = mask + (size_t)seg * max_seg_len * max_cb;
  const float4* b4 = reinterpret_cast<const float4*>(boxes) + beg;

  __shared__ float4 col_boxes[kNmsTile];
  if (threadIdx.x < col_size) col_boxes[threadIdx.x] = b4[col_t * kNmsTile + threadIdx.x];
  __syncthreads();
  if (threadIdx.x < row_size) {
    const int cur = row_t * kNmsTile + threadIdx.x;
    const float4 me = b4[cur];
    unsigned long long t = 0;
    const int start = (row_t == col_t) ? threadIdx.x + 1 : 0;
    for (int i = start; i < col_size; ++i)
      if (dev_iou(me, col_boxes[i]) > thresh) t |= 1ULL << i;
    seg_mask[(size_t)cur * max_cb + col_t] = t;
  }
}

// grid (S), block kSweepThreads.  keep_out [S, max_seg_len], keep_cnt [S]
constexpr int kSweepThreads = 256;
__global__ void __launch_bounds__(kSweepThreads)
nms_sweep_kernel(const int* __restrict__ seg_offsets, int max_seg_len,
                 const unsigned long long* __restrict__ mask, int* __restrict__ keep_out,
                 int* __restrict__ keep_cnt) {
  extern __shared__ unsigned long long removed[];  // [col_blocks]
  __shared__ unsigned long long diag[kNmsTile];
  __shared__ unsigned long long kept_word;
  __shared__ int count;

  const int seg = blockIdx.x;
  const int n = min(seg_offsets[seg + 1] - seg_offsets[seg], max_seg_len);
  const int cb = ceil_div(n, kNmsTile);
  const int max_cb = ceil_div(max_seg_len, kNmsTile);
  const unsigned long long* seg_mask = mask + (size_t)seg * max_seg_len * max_cb;
  int* keep = keep_out + (size_t)seg * max_seg_len;

  for (int j = threadIdx.x; j < cb; j += blockDim.x) removed[j] = 0ULL;
  if (threadIdx.x == 0) count = 0;
  __syncthreads();

  for (int b = 0; b < cb; ++b) {
    const int bsize = min(n - b * kNmsTile, kNmsTile);
    if (threadIdx.x < kNmsTile)
      diag[threadIdx.x] = threadIdx.x < bsize
                              ? seg_mask[(size_t)(b * kNmsTile + threadIdx.x) * max_cb + b]
                              : 0ULL;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long cur = removed[b], K = 0ULL;
      unsigned long long d[kNmsTile];
#pragma unroll
      for (int t = 0; t < kNmsTile; ++t) d[t] = diag[t];     // 64 independent LDS, then a pure ALU chain
#pragma unroll
      for (int t = 0; t < kNmsTile; ++t) {
        const bool take = (t < bsize) && !((cur >> t) & 1ULL);
        K |= take ? (1ULL << t) : 0ULL;
        cur |= take ? d[t] : 0ULL;
      }
      kept_word = K;
    }
    __syncthreads();
    const unsigned long long K = kept_word;
    const int base_cnt = count;
    if (threadIdx.x < kNmsTile && ((K >> threadIdx.x) & 1ULL)) {
      const int pos = base_cnt + __popcll(K & ((1ULL << threadIdx.x) - 1ULL));
      keep[pos] = b * kNmsTile + threadIdx.x;
    }
    // OR the kept rows into the running removed words of the later blocks.  Loads are issued in
    // predicated batches of 8 so that they overlap (a data-dependent `while` over the set bits
    // would serialise one L2 round trip per kept box).
    for (int j = b + 1 + threadIdx.x; j < cb; j += blockDim.x) {
      unsigned long long acc = removed[j];
      const unsigned long long* col = seg_mask + (size_t)(b * kNmsTile) * max_cb + j;
#pragma unroll 1
      for (int t0 = 0; t0 < kNmsTile; t0 += 8) {
        const unsigned int bits = (unsigned int)((K >> t0) & 0xffULL);
        if (bits == 0) continue;
        unsigned long long v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = ((bits >> u) & 1u) ? col[(size_t)(t0 + u) * max_cb] : 0ULL;
        acc |= (v[0] | v[1]) | (v[2] | v[3]) | (v[4] | v[5]) | (v[6] | v[7]);
      }
      removed[j] = acc;
    }
    __syncthreads();
    if (threadIdx.x == 0) count = base_cnt + __popcll(K);
    // next iteration's first __syncthreads orders the count update before its readers
  }
  __syncthreads();
  if (threadIdx.x == 0) keep_cnt[seg] = count;
}

// Same sweep with the segment's whole bitmask staged in shared memory first (one coalesced cp.async pass):
// for segments of up to ~1200 boxes (every NMS of the UPSNet path: 1000 proposals per level / per class) the
// 64 dependent steps of a diagonal word and the kept-row ORs then run at shared-memory latency instead of one
// L2 round trip per batch of rows.  grid (S), block kSweepSmemThreads, dynamic smem = (max_seg_len + 1) * cb * 8.
constexpr int kSweepSmemThreads = 1024;
__global__ void __launch_bounds__(kSweepSmemThreads)
nms_sweep_smem_kernel(const int* __restrict__ seg_offsets, int max_seg_len,
                      const unsigned long long* __restrict__ mask, int* __restrict__ keep_out,
                      int* __restrict__ keep_cnt) {
  extern __shared__ __align__(16) unsigned long long sm_mask[];   // [n][cb] then removed[cb]
  __shared__ unsigned long long kept_word;
  __shared__ int count;
  const int seg = blockIdx.x;
  const int n = min(seg_offsets[seg + 1] - seg_offsets[seg], max_seg_len);
  const int cb = ceil_div(n, kNmsTile);
  const int max_cb = ceil_div(max_seg_len, kNmsTile);
  const unsigned long long* seg_mask = mask + (size_t)seg * max_seg_len * max_cb;
  int* keep = keep_out + (size_t)seg * max_seg_len;
  unsigned long long* removed = sm_mask + (size_t)n * cb;
  // stage rows [0,n) x words [row/64, cb): the mask kernel only writes the upper-triangular tiles
  for (int e = threadIdx.x; e < n * cb; e += kSweepSmemThreads) {
    const int r = e / cb, j = e - r * cb;
    if (j >= r / kNmsTile) {
      const unsigned int dst = (unsigned int)__cvta_generic_to_shared(sm_mask + e);
      asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(seg_mask + (size_t)r * max_cb + j) : "memory");
    }
  }
  for (int j = threadIdx.x; j < cb; j += kSweepSmemThreads) removed[j] = 0ULL;
  if (threadIdx.x == 0) count = 0;
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
  __syncthreads();

  for (int b = 0; b < cb; ++b) {
    const int bsize = min(n - b * kNmsTile, kNmsTile);
    if (threadIdx.x == 0) {
      unsigned long long cur = removed[b], K = 0ULL;
      unsigned long long d[kNmsTile];
#pragma unroll
      for (int t = 0; t < kNmsTile; ++t) d[t] = t < bsize ? sm_mask[(size_t)(b * kNmsTile + t) * cb + b] : 0ULL;
#pragma unroll
      for (int t = 0; t < kNmsTile; ++t) {
        const bool take = (t < bsize) && !((cur >> t) & 1ULL);
        K |= take ? (1ULL << t) : 0ULL;
        cur |= take ? d[t] : 0ULL;
      }
      kept_word = K;
    }
    __syncthreads();
    const unsigned long long K = kept_word;
    const int base_cnt = count;
    if (threadIdx.x < kNmsTile && ((K >> threadIdx.x) & 1ULL))
      keep[base_cnt + __popcll(K & ((1ULL << threadIdx.x) - 1ULL))] = b * kNmsTile + threadIdx.x;
    // kept rows -> removed words of the later blocks: 16 lanes per word column, 4 rows each, xor-shuffle OR
    {
      const int lane16 = threadIdx.x & 15, warp2 = (threadIdx.x >> 5) * 2, sub = (threadIdx.x >> 4) & 1;
      for (int j0 = b + 1 + warp2; j0 < cb; j0 += kSweepSmemThreads / 16) {   // warp-uniform trip count
        const int j = j0 + sub;
        const bool ok = j < cb;
        unsigned long long acc = 0ULL;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int t = lane16 * 4 + u;
          if (ok && ((K >> t) & 1ULL)) acc |= sm_mask[(size_t)(b * kNmsTile + t) * cb + j];
        }
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) acc |= __shfl_xor_sync(0xffffffffu, acc, o, 16);
        if (ok && lane16 == 0) removed[j] |= acc;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) count = base_cnt + __popcll(K);
  }
  __syncthreads();
  if (threadIdx.x == 0) keep_cnt[seg] = count;
}

static size_t nms_mask_bytes(int S, int max_seg_len) {
  return (size_t)S * max_seg_len * ceil_div(max_seg_len, kNmsTile) * sizeof(unsigned long long);
}

}  // namespace ups

extern "C" int upsnet_nms_workspace_bytes(int S, int max_seg_len, size_t* bytes) {
  if (!bytes || S <= 0 || max_seg_len <= 0 || max_seg_len > ups::kNmsMaxSeg) return UPSNET_E_BADARG;
  *bytes = ups::nms_mask_bytes(S, max_seg_len);
  return 0;
}

extern "C" int upsnet_nms_segmented(const float* boxes, const int* seg_offsets, int S,
                                    int max_seg_len, float thresh, int* keep_out, int* keep_cnt,
                                    void* workspace, size_t workspace_bytes, void* stream) {
  using namespace ups;
  if (!boxes || !seg_offsets || !keep_out || !keep_cnt || !workspace) return UPSNET_E_BADARG;
  if (S <= 0 || max_seg_len <= 0 || max_seg_len > kNmsMaxSeg) return UPSNET_E_BADARG;
  if (((uintptr_t)boxes & 15) != 0) return UPSNET_E_BADARG;  // float4 loads
  if (workspace_bytes < nms_mask_bytes(S, max_seg_len)) return UPSNET_E_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const int tiles = ceil_div(max_seg_len, kNmsTile);
  if (tiles > 65535 || S > 65535) return UPSNET_E_UNSUPPORTED;
  dim3 grid(tiles, tiles, S);
  nms_mask_kernel<<<grid, kNmsTile, 0, st>>>(boxes, seg_offsets, max_seg_len, thresh,
                                             (unsigned long long*)workspace);
  UPS_CHECK_LAUNCH();
  const size_t smem_all = ((size_t)max_seg_len + 1) * tiles * sizeof(unsigned long long);
  if (smem_all <= 200 * 1024) {   // whole per-segment bitmask fits in shared memory
    static ups::PerDeviceOnce configured;
    if (configured.need()) {
      UPS_CUDA(cudaFuncSetAttribute(nms_sweep_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    }
    nms_sweep_smem_kernel<<<S, kSweepSmemThreads, smem_all, st>>>(seg_offsets, max_seg_len,
                                                                  (const unsigned long long*)workspace, keep_out, keep_cnt);
    UPS_CHECK_LAUNCH();
    return 0;
  }
  const size_t smem = (size_t)tiles * sizeof(unsigned long long);
  nms_sweep_kernel<<<S, kSweepThreads, smem, st>>>(seg_offsets, max_seg_len,
                                                   (const unsigned long long*)workspace, keep_out,
                                                   keep_cnt);
  UPS_CHECK_LAUNCH();
  return 0;
}

// Drop-in for the reference's `_nms` (nms/gpu_nms.hpp:14): host pointers, allocates and
// synchronises exactly like the reference does, but sweeps on the device.
extern "C" int upsnet_nms_host(int* keep_out, int* num_out, const float* boxes_host,
                               int boxes_num, int boxes_dim, float thresh, int device_id) {
  using namespace ups;
  if (!keep_out || !num_out || (!boxes_host && boxes_num > 0) || boxes_dim < 4) return UPSNET_E_BADARG;
  if (boxes_num > kNmsMaxSeg) return UPSNET_E_UNSUPPORTED;
  *num_out = 0;
  if (boxes_num <= 0) return 0;
  int prev = 0;
  UPS_CUDA(cudaGetDevice(&prev));
  if (prev != device_id) UPS_CUDA(cudaSetDevice(device_id));
  const int n = boxes_num;
  float* hb = (float*)malloc(sizeof(float) * 4 * n);
  if (!hb) return UPSNET_E_BADARG;
  for (int i = 0; i < n; ++i)
    for (int k = 0; k < 4; ++k) hb[i * 4 + k] = boxes_host[(size_t)i * boxes_dim + k];
  const size_t wbytes = nms_mask_bytes(1, n);
  char* dev = nullptr;
  const size_t off_boxes = 0, off_seg = align_up(sizeof(float) * 4 * n, 256);
  const size_t off_keep = off_seg + 256, off_cnt = off_keep + align_up(sizeof(int) * n, 256);
  const size_t off_ws = off_cnt + 256;
  int rc = 0;
  cudaError_t e = cudaMalloc(&dev, off_ws + wbytes);
  if (e != cudaSuccess) { free(hb); return (int)e; }
  const int seg[2] = {0, n};
  e = cudaMemcpy(dev + off_boxes, hb, sizeof(float) * 4 * n, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(dev + off_seg, seg, sizeof(seg), cudaMemcpyHostToDevice);
  if (e == cudaSuccess)
    rc = upsnet_nms_segmented((const float*)(dev + off_boxes), (const int*)(dev + off_seg), 1, n,
                              thresh, (int*)(dev + off_keep), (int*)(dev + off_cnt), dev + off_ws,
                              wbytes, nullptr);
  if (e == cudaSuccess && rc == 0) e = cudaMemcpy(num_out, dev + off_cnt, sizeof(int), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess && rc == 0)
    e = cudaMemcpy(keep_out, dev + off_keep, sizeof(int) * (*num_out), cudaMemcpyDeviceToHost);
  cudaFree(dev);
  free(hb);
  if (prev != device_id) cudaSetDevice(prev);
  if (rc != 0) return rc;
  return (int)e;
}
