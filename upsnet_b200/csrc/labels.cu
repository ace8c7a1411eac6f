// labels.cu -- the panoptic training labels of one image (the label block of the reference's Cityscapes / COCO loaders
// and collate / gt_list_to_blob): seg_gt, seg_gt_4x and seg_roi_gt as gathers from the uint8 label map through host-built
// cv2 INTER_NEAREST index tables, and mask_gt by Pillow's polygon fill evaluated only on the canvas rows and columns the
// two nearest resizes sample.  No full-resolution instance image exists.  See include/upsnet_b200.h for the contract.
//
// Determinism: every output element has one owner thread; there is no atomic in this file.
#include "common.cuh"

namespace ups {
namespace {

constexpr int kLbThreads = 256;
constexpr int kLbWarps = 2;                        // mask_gt: one output row per warp
constexpr int kLbMaxX = UPSNET_LABELS_MAX_POLY_VERTS * 2;   // intersections of one polygon on one row
constexpr int kLbMaxSpans = UPSNET_LABELS_MAX_OBJ_VERTS;    // spans of one instance on one row

// seg_gt / seg_gt_4x / seg_roi_gt: out[i, y, x] = label[rows[i * nr + y], cols[i * nc + x]], 255 where a table is -1
__global__ void lb_gather_kernel(const unsigned char* __restrict__ label, int w0, const int* __restrict__ rows,
                                 const int* __restrict__ cols, int nr, int nc, long long total, int64_t* __restrict__ out) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long plane = (long long)nr * nc;
    const int i = (int)(e / plane);
    const int rem = (int)(e - (long long)i * plane);
    const int y = rem / nc, x = rem - y * nc;
    const int r = rows[(long long)i * nr + y], c = cols[(long long)i * nc + x];
    out[e] = (r < 0 || c < 0) ? 255 : (int64_t)label[(long long)r * w0 + c];
  }
}

__device__ __forceinline__ float lb_x_at(int x0, int y0, float dx, int y) {
  return __fadd_rn(__fmul_rn(__int2float_rn(y - y0), dx), __int2float_rn(x0));
}

// Pillow's ROUND_UP / ROUND_DOWN (Draw.c): by magnitude, float32 for x >= 0, double for x < 0
__device__ __forceinline__ int lb_round_up(float x) {
  return x >= 0.f ? (int)floorf(__fadd_rn(x, 0.5f)) : -(int)floor((double)fabsf(x) + 0.5);
}
__device__ __forceinline__ int lb_round_down(float x) {
  return x >= 0.f ? (int)ceilf(__fsub_rn(x, 0.5f)) : -(int)ceil((double)fabsf(x) - 0.5);
}

struct LbEdge {
  int x0, y0, x1, y1;
};

__device__ __forceinline__ LbEdge lb_edge(const int* v, int n, int i) {
  const int j = i + 1 == n ? 0 : i + 1;
  return LbEdge{v[2 * i], v[2 * i + 1], v[2 * j], v[2 * j + 1]};
}

// The spans polygon_generic sets on canvas row Y for one polygon of n truncated vertices (tests/label_oracle.py states
// the rule).  Appends to spans; xx is this warp's scratch.  Runs on one thread.
__device__ int lb_polygon_row(const int* v, int n, int Y, float* xx, int2* spans, int ns) {
  int ymax = v[1];
  for (int i = 0; i < n; ++i) {
    const LbEdge e = lb_edge(v, n, i);
    ymax = max(ymax, e.y0);
    if (e.y0 == e.y1 && e.y0 == Y) spans[ns++] = make_int2(min(e.x0, e.x1), max(e.x0, e.x1));
  }
  int j = 0;
  for (int i = 0; i < n; ++i) {
    const LbEdge e = lb_edge(v, n, i);
    if (e.y0 == e.y1) continue;                 // horizontal, or both ends in one pixel
    const int emin = min(e.y0, e.y1), emax = max(e.y0, e.y1);
    if (Y < emin || Y > emax) continue;
    const float dx = __fdiv_rn(__int2float_rn(e.x1 - e.x0), __int2float_rn(e.y1 - e.y0));
    float x = lb_x_at(e.x0, e.y0, dx, Y);
    if (Y == emax && Y < ymax) {
      xx[j++] = x;
      xx[j++] = x;
      continue;
    }
    if ((Y == emin || Y == emax) && dx != 0.f) {
      const int r = Y == emax ? Y - 1 : Y + 1;
      const float rx = roundf(x);
      for (int k = 0; k < i; ++k) {
        const LbEdge o = lb_edge(v, n, k);
        if (o.y0 == o.y1) continue;
        const int omin = min(o.y0, o.y1), omax = max(o.y0, o.y1);
        if (Y != omin && Y != omax) continue;
        const float odx = __fdiv_rn(__int2float_rn(o.x1 - o.x0), __int2float_rn(o.y1 - o.y0));
        if (odx == 0.f || roundf(lb_x_at(o.x0, o.y0, odx, Y)) != rx) continue;
        if (r < omin || r > omax) continue;
        const float a = lb_x_at(e.x0, e.y0, dx, r), b = lb_x_at(o.x0, o.y0, odx, r);
        if (x > __fadd_rn(a, 1.f) && x > __fadd_rn(b, 1.f))
          x = __fadd_rn(roundf(fmaxf(a, b)), 1.f);
        else if (x < __fsub_rn(a, 1.f) && x < __fsub_rn(b, 1.f))
          x = __fsub_rn(roundf(fminf(a, b)), 1.f);
        break;
      }
    }
    xx[j++] = x;
  }
  for (int a = 1; a < j; ++a) {                 // insertion sort: a row meets few edges
    const float t = xx[a];
    int b = a - 1;
    while (b >= 0 && xx[b] > t) {
      xx[b + 1] = xx[b];
      --b;
    }
    xx[b + 1] = t;
  }
  for (int a = 1; a < j; a += 2) {
    const int s = lb_round_up(xx[a - 1]), t = lb_round_down(xx[a]);
    if (t >= s) spans[ns++] = make_int2(s, t);
  }
  return ns;
}

// mask_gt: one CTA per (instance, pair of output rows), one warp per row
template <typename T>
__global__ void __launch_bounds__(kLbWarps * 32) lb_mask_kernel(const int* __restrict__ m_rows, int Hm,
                                                                const int* __restrict__ m_cols, int Wm,
                                                                const int* __restrict__ obj_poly,
                                                                const int* __restrict__ poly_vert,
                                                                const int* __restrict__ verts,
                                                                const int* __restrict__ obj_yrange, T* __restrict__ out) {
  __shared__ float s_xx[kLbWarps][kLbMaxX];
  __shared__ int2 s_spans[kLbWarps][kLbMaxSpans];
  __shared__ int s_ns[kLbWarps];
  const int g = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int y = blockIdx.y * kLbWarps + warp;
  if (y >= Hm) return;
  T* row = out + ((long long)g * Hm + y) * Wm;
  const int Y = m_rows[y];
  if (Y < 0) {
    for (int x = lane; x < Wm; x += 32) row[x] = (T)255;
    return;
  }
  if (Y < obj_yrange[2 * g] || Y > obj_yrange[2 * g + 1]) {     // outside the instance's integer rows: no edge looked at
    for (int x = lane; x < Wm; x += 32) row[x] = m_cols[x] < 0 ? (T)255 : (T)0;
    return;
  }
  if (lane == 0) {
    int ns = 0;
    for (int p = obj_poly[g]; p < obj_poly[g + 1]; ++p)
      ns = lb_polygon_row(verts + 2 * poly_vert[p], poly_vert[p + 1] - poly_vert[p], Y, s_xx[warp], s_spans[warp], ns);
    s_ns[warp] = ns;
  }
  __syncwarp();
  const int ns = s_ns[warp];
  for (int x = lane; x < Wm; x += 32) {
    const int X = m_cols[x];
    T v = (T)255;
    if (X >= 0) {
      v = (T)0;
      for (int s = 0; s < ns; ++s) {
        const int2 sp = s_spans[warp][s];
        if (X >= sp.x && X <= sp.y) {
          v = (T)1;
          break;
        }
      }
    }
    row[x] = v;
  }
}

int lb_gather(const unsigned char* label, int w0, const int* rows, const int* cols, int nr, int nc, int n, int64_t* out,
              cudaStream_t st) {
  const long long total = (long long)n * nr * nc;
  if (total == 0) return 0;
  const int blocks = (int)std::min<long long>(ceil_div(total, (long long)kLbThreads), 132LL * 16);
  lb_gather_kernel<<<blocks, kLbThreads, 0, st>>>(label, w0, rows, cols, nr, nc, total, out);
  UPS_CHECK_LAUNCH();
  return 0;
}

}  // namespace
}  // namespace ups

extern "C" int upsnet_training_labels(const unsigned char* label, int h0, int w0, const int* seg_rows, int Hs,
                                      const int* seg_cols, int Ws, int64_t* seg_gt, const int* q_rows, int Hq,
                                      const int* q_cols, int Wq, int64_t* seg_gt_4x, const int* m_rows, int Hm,
                                      const int* m_cols, int Wm, const int* obj_poly, const int* poly_vert,
                                      const int* verts, const int* obj_yrange, int G, int max_poly_verts,
                                      int max_obj_verts, void* mask_gt, int mask_gt_is_int64, const int* roi_rows,
                                      const int* roi_cols, int n_roi, int M, int64_t* seg_roi_gt, void* stream) {
  using namespace ups;
  if (!label || h0 <= 0 || w0 <= 0 || !seg_rows || !seg_cols || !seg_gt || Hs <= 0 || Ws <= 0 || !q_rows || !q_cols ||
      !seg_gt_4x || Hq <= 0 || Wq <= 0 || G < 0 || n_roi < 0)
    return UPSNET_E_BADARG;
  if (G > 0 && (!m_rows || !m_cols || Hm <= 0 || Wm <= 0 || !obj_poly || !poly_vert || !verts || !obj_yrange || !mask_gt))
    return UPSNET_E_BADARG;
  if (n_roi > 0 && (!roi_rows || !roi_cols || !seg_roi_gt || M <= 0)) return UPSNET_E_BADARG;
  if (max_poly_verts > UPSNET_LABELS_MAX_POLY_VERTS || max_obj_verts > UPSNET_LABELS_MAX_OBJ_VERTS ||
      G > UPSNET_LABELS_MAX_G || (size_t)h0 * w0 >= (1ull << 31) || (size_t)Hs * Ws >= (1ull << 31) ||
      (size_t)Hm * Wm >= (1ull << 31) || ceil_div(Hm, kLbWarps) > 65535)
    return UPSNET_E_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = lb_gather(label, w0, seg_rows, seg_cols, Hs, Ws, 1, seg_gt, st);
  if (!rc) rc = lb_gather(label, w0, q_rows, q_cols, Hq, Wq, 1, seg_gt_4x, st);
  if (!rc && n_roi > 0) rc = lb_gather(label, w0, roi_rows, roi_cols, M, M, n_roi, seg_roi_gt, st);
  if (rc) return rc;
  if (G > 0) {
    const dim3 grid(G, ceil_div(Hm, kLbWarps));
    if (mask_gt_is_int64)
      lb_mask_kernel<int64_t><<<grid, kLbWarps * 32, 0, st>>>(m_rows, Hm, m_cols, Wm, obj_poly, poly_vert, verts,
                                                             obj_yrange, (int64_t*)mask_gt);
    else
      lb_mask_kernel<unsigned char><<<grid, kLbWarps * 32, 0, st>>>(m_rows, Hm, m_cols, Wm, obj_poly, poly_vert, verts,
                                                                   obj_yrange, (unsigned char*)mask_gt);
    UPS_CHECK_LAUNCH();
  }
  return 0;
}
