// impost.cu -- row f4 of SURVEY section 8: the instance-mask post-processing of the test loop on the device.
//
// Reference: upsnet_end2end_test.py:95-152 `im_post` -- per detection: expand the box by (M+2)/M (bbox_transform.py:365-381
// expand_boxes, float32 arithmetic, then .astype(np.int32) = truncation), zero-pad the M x M mask probability of the
// predicted class to (M+2) x (M+2), cv2.resize it (INTER_LINEAR) to the box size, threshold > 0.5, paste it into an
// [H, W] uint8 image clipped at the borders and RLE-encode that image with pycocotools.mask.encode (column-major run
// lengths, starting with the zeros run).  The reference does this on the host with numpy + cv2 + pycocotools for every
// detection of every image (after a D2H copy of all mask probabilities).
//
// Here one CTA per detection never materialises the image: every thread walks whole COLUMNS of the detection's clipped
// window, evaluates the resized mask (OpenCV's documented formula in un-fused fp32, the same rule as the panoptic head's
// MaskRemoval: SURVEY A.5) and counts run starts / ends; a block scan turns the per-column counts into offsets, a second
// walk writes the absolute column-major positions of every run boundary and a last pass differences them into the COCO
// counts.  Runs that continue from the last row of one column into the first row of the next (only possible when the
// window spans the full image height) are merged exactly as pycocotools' linear scan does.
// Roofline: none worth naming (KBs in, KBs out; ~3 evaluations of the 4-tap blend per window pixel).
#include <cstdint>

#include "common.cuh"

namespace ups {

constexpr int kPostThreads = 256;
constexpr int kPostMaxM = 30;          // padded mask side (M + 2), M <= 28
constexpr int kPostMaxCols = 2048;     // window columns whose counts live in shared memory
constexpr int kPostMaxRows = 2048;     // window rows whose resize coefficients live in shared memory

struct PostBox { int bx0, by0, w, h, x0, x1, y0, y1; };

// bbox_transform.py:365-381 + upsnet_end2end_test.py:104-105,120-133 (float32 arithmetic, int32 truncation)
__device__ __forceinline__ PostBox post_box(const float* __restrict__ b, float scale, int H, int W) {
  const float wh = __fmul_rn(__fmul_rn(__fsub_rn(b[2], b[0]), 0.5f), scale);
  const float hh = __fmul_rn(__fmul_rn(__fsub_rn(b[3], b[1]), 0.5f), scale);
  const float xc = __fmul_rn(__fadd_rn(b[2], b[0]), 0.5f), yc = __fmul_rn(__fadd_rn(b[3], b[1]), 0.5f);
  PostBox r;
  r.bx0 = (int)__fsub_rn(xc, wh); r.by0 = (int)__fsub_rn(yc, hh);
  const int bx1 = (int)__fadd_rn(xc, wh), by1 = (int)__fadd_rn(yc, hh);
  r.w = max(bx1 - r.bx0 + 1, 1); r.h = max(by1 - r.by0 + 1, 1);
  r.x0 = max(r.bx0, 0); r.x1 = min(bx1 + 1, W); r.y0 = max(r.by0, 0); r.y1 = min(by1 + 1, H);
  // the reference pastes mask[(y0 - by0):(y1 - by0), (x0 - bx0):(x1 - bx0)] of the (h, w) resize: never beyond its extent
  r.x1 = min(r.x1, r.bx0 + r.w); r.y1 = min(r.y1, r.by0 + r.h);
  return r;
}

// cv2.resize INTER_LINEAR coefficients for a float32 image (source size S, destination size n): float64 scale, float32
// coordinate; columns clamp the tap and zero the fraction at both borders, rows clamp the taps only
__device__ __forceinline__ void post_coef(int d, int n, int S, bool is_x, int& s, float& f) {
  const double scale = __ddiv_rn((double)S, (double)n);
  float fv = (float)__dadd_rn(__dmul_rn((double)d + 0.5, scale), -0.5);
  int sv = (int)floorf(fv);
  fv = __fsub_rn(fv, (float)sv);
  if (is_x) {
    if (sv < 0) { sv = 0; fv = 0.f; }
    if (sv >= S - 1) { sv = S - 1; fv = 0.f; }
  }
  s = sv; f = fv;
}

struct PostCol { int sx, sx1; float a0, a1; };

// value of the resized mask at (column coefficients c, row coefficients (sy, fy)) > 0.5
__device__ __forceinline__ bool post_bit(const float* __restrict__ P, int S, const PostCol& c, int sy, float fy) {
  const int y0 = min(max(sy, 0), S - 1), y1 = min(max(sy + 1, 0), S - 1);
  const float b0 = __fsub_rn(1.f, fy);
  const float h0 = __fadd_rn(__fmul_rn(P[y0 * S + c.sx], c.a0), __fmul_rn(P[y0 * S + c.sx1], c.a1));
  const float h1 = __fadd_rn(__fmul_rn(P[y1 * S + c.sx], c.a0), __fmul_rn(P[y1 * S + c.sx1], c.a1));
  return __fadd_rn(__fmul_rn(h0, b0), __fmul_rn(h1, fy)) > 0.5f;
}

__device__ __forceinline__ PostCol post_col(int dx, int w, int S) {
  PostCol c; float fx;
  post_coef(dx, w, S, true, c.sx, fx);
  c.sx1 = min(c.sx + 1, S - 1);
  c.a0 = __fsub_rn(1.f, fx); c.a1 = fx;
  return c;
}

// block-wide exclusive scan of v[0..n) in shared memory (n <= kPostMaxCols), returns the total
__device__ int post_scan(int* v, int n, int* s_part) {
  const int per = (n + kPostThreads - 1) / kPostThreads;
  const int lo = min((int)threadIdx.x * per, n), hi = min(lo + per, n);
  int sum = 0;
  for (int i = lo; i < hi; ++i) sum += v[i];
  s_part[threadIdx.x] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int t = 0; t < kPostThreads; ++t) { const int x = s_part[t]; s_part[t] = acc; acc += x; }
    s_part[kPostThreads] = acc;
  }
  __syncthreads();
  int acc = s_part[threadIdx.x];
  for (int i = lo; i < hi; ++i) { const int x = v[i]; v[i] = acc; acc += x; }
  __syncthreads();
  return s_part[kPostThreads];
}

// grid = n detections.  counts [n][cap] uint32, run_len [n] (number of counts, 0 for d >= n_dev), overflow[0] |= 1 when a
// detection needs more than cap counts (its run_len is then the needed size, its counts are truncated).
__global__ void __launch_bounds__(kPostThreads)
im_post_rle_kernel(const float* __restrict__ mask_probs, int C, int M, const float* __restrict__ boxes,
                   const int64_t* __restrict__ cls_inds, int n, const int* __restrict__ n_dev, int H, int W,
                   uint32_t* __restrict__ counts, long long* __restrict__ pos_ws, int cap, int* __restrict__ run_len,
                   int* __restrict__ overflow) {
  __shared__ float P[kPostMaxM * kPostMaxM];
  __shared__ int s_starts[kPostMaxCols], s_ends[kPostMaxCols];
  __shared__ int s_part[kPostThreads + 1];
  __shared__ short s_sy[kPostMaxRows];
  __shared__ float s_fy[kPostMaxRows];
  const int d = blockIdx.x;
  const int live = n_dev ? min(*n_dev, n) : n;
  if (d >= live) { if (threadIdx.x == 0) run_len[d] = 0; return; }
  const int S = M + 2;
  const int cls = C > 1 ? (int)cls_inds[d] : 0;
  for (int t = threadIdx.x; t < S * S; t += kPostThreads) {
    const int y = t / S, x = t - y * S;
    float v = 0.f;
    if (y >= 1 && y <= M && x >= 1 && x <= M) v = __ldg(mask_probs + (((size_t)d * C + cls) * M + (y - 1)) * M + (x - 1));
    P[t] = v;
  }
  const float scale = (float)(((double)M + 2.0) / (double)M);       // python float -> float32 in `w_half *= scale`
  const PostBox b = post_box(boxes + (size_t)d * 4, scale, H, W);
  const int ncol = max(b.x1 - b.x0, 0), nrow = max(b.y1 - b.y0, 0);
  uint32_t* out = counts + (size_t)d * cap;
  long long* pos = pos_ws + (size_t)d * cap;
  const long long HW = (long long)H * W;
  __syncthreads();
  if (ncol == 0 || nrow == 0) {                  // empty paste: one run of zeros
    if (threadIdx.x == 0) { out[0] = (uint32_t)HW; run_len[d] = 1; }
    return;
  }
  const bool wrap = b.y0 == 0 && b.y1 == H;      // only then can a run continue from one column into the next
  for (int t = threadIdx.x; t < nrow; t += kPostThreads) {     // row coefficients of the window, once per detection
    int sy; float fy;
    post_coef(b.y0 + t - b.by0, b.h, S, false, sy, fy);
    s_sy[t] = (short)sy; s_fy[t] = fy;
  }
  __syncthreads();
  const int rlast = nrow - 1;                    // window row of image row H - 1 when wrap
  // ---- pass 1: run starts / ends per column ----
  for (int c = threadIdx.x; c < ncol; c += kPostThreads) {
    const int x = b.x0 + c;
    const PostCol pc = post_col(x - b.bx0, b.w, S);
    bool prev = false;
    if (wrap && c > 0) prev = post_bit(P, S, post_col(x - 1 - b.bx0, b.w, S), s_sy[rlast], s_fy[rlast]);
    int ns = 0, ne = 0;
    for (int y = b.y0; y < b.y1; ++y) {
      const bool bit = post_bit(P, S, pc, s_sy[y - b.y0], s_fy[y - b.y0]);
      ns += (bit && !prev); ne += (!bit && prev);
      prev = bit;
    }
    if (prev) {                                  // run reaches the bottom of the window
      bool cont = false;
      if (wrap && c + 1 < ncol) cont = post_bit(P, S, post_col(x + 1 - b.bx0, b.w, S), s_sy[0], s_fy[0]);
      if (!cont) ++ne;
    }
    if (c < kPostMaxCols) { s_starts[c] = ns; s_ends[c] = ne; }
  }
  __syncthreads();
  const int runs = post_scan(s_starts, ncol, s_part);
  const int runs_e = post_scan(s_ends, ncol, s_part);
  (void)runs_e;                                  // == runs
  // ---- pass 2: absolute column-major positions of the boundaries: pos[2k] = start, pos[2k+1] = end (exclusive) ----
  for (int c = threadIdx.x; c < ncol; c += kPostThreads) {
    const int x = b.x0 + c;
    const PostCol pc = post_col(x - b.bx0, b.w, S);
    bool prev = false;
    if (wrap && c > 0) prev = post_bit(P, S, post_col(x - 1 - b.bx0, b.w, S), s_sy[rlast], s_fy[rlast]);
    int ks = s_starts[c], ke = s_ends[c];
    const long long colbase = (long long)x * H;
    for (int y = b.y0; y < b.y1; ++y) {
      const bool bit = post_bit(P, S, pc, s_sy[y - b.y0], s_fy[y - b.y0]);
      if (bit && !prev) { if (2 * ks < cap) pos[2 * ks] = colbase + y; ++ks; }
      if (!bit && prev) { if (2 * ke + 1 < cap) pos[2 * ke + 1] = colbase + y; ++ke; }
      prev = bit;
    }
    if (prev) {
      bool cont = false;
      if (wrap && c + 1 < ncol) cont = post_bit(P, S, post_col(x + 1 - b.bx0, b.w, S), s_sy[0], s_fy[0]);
      if (!cont) { if (2 * ke + 1 < cap) pos[2 * ke + 1] = colbase + b.y1; ++ke; }
    }
  }
  __syncthreads();
  // ---- pass 3: counts = differences of consecutive boundaries (+ the trailing zeros run) ----
  long long last_end = 0;
  if (runs > 0 && 2 * runs - 1 < cap) last_end = pos[2 * runs - 1];
  const bool tail = runs == 0 || last_end < HW;
  const int m = 2 * runs + (tail ? 1 : 0);
  for (int j = threadIdx.x; j < min(2 * runs, cap); j += kPostThreads)
    out[j] = (uint32_t)(pos[j] - (j > 0 ? pos[j - 1] : 0ll));
  if (threadIdx.x == 0) {
    if (tail && m - 1 < cap) out[m - 1] = (uint32_t)(HW - (runs > 0 ? last_end : 0ll));
    run_len[d] = m;
    if (m > cap) atomicOr(overflow, 1);
  }
}

// the run boundaries of every detection, [n][cap]
inline size_t im_post_layout(int n, int cap, void* base, long long** pos) {
  WsCarve c(base);
  *pos = c.take<long long>((size_t)(n > 0 ? n : 1) * cap);
  return c.bytes();
}

}  // namespace ups

extern "C" int upsnet_im_post_workspace_bytes(int n, int cap, size_t* bytes) {
  if (!bytes || n < 0 || cap < 2) return UPSNET_E_BADARG;
  long long* pos;
  *bytes = ups::im_post_layout(n, cap, nullptr, &pos);
  return 0;
}

extern "C" int upsnet_im_post_rle(const float* mask_probs, int C, int M, const float* boxes, const int64_t* cls_inds, int n,
                                  const int* n_dev, int H, int W, uint32_t* counts, int cap, int* run_len, int* overflow,
                                  void* workspace, size_t workspace_bytes, void* stream) {
  using namespace ups;
  if (!mask_probs || !boxes || !cls_inds || !counts || !run_len || !overflow || !workspace) return UPSNET_E_BADARG;
  if (n < 0 || C < 1 || M < 1 || H <= 0 || W <= 0 || cap < 2) return UPSNET_E_BADARG;
  if (M + 2 > kPostMaxM || W > kPostMaxCols || H > kPostMaxRows) return UPSNET_E_UNSUPPORTED;
  long long* pos;
  if (workspace_bytes < im_post_layout(n, cap, workspace, &pos)) return UPSNET_E_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  UPS_CUDA(cudaMemsetAsync(overflow, 0, sizeof(int), st));
  if (n == 0) return 0;
  im_post_rle_kernel<<<n, kPostThreads, 0, st>>>(mask_probs, C, M, boxes, cls_inds, n, n_dev, H, W, counts, pos, cap, run_len,
                                                 overflow);
  UPS_CHECK_LAUNCH();
  return 0;
}
