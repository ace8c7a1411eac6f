// proposal_target.cu -- Mask R-CNN proposal targets of one image (operators/modules/proposal_mask_target.py:37-62):
// add_proposals (dataset/json_dataset.py:335-348, 454-516, 538-556), sample_rois (bbox/sample_rois.py:51-176) and
// add_mask_rcnn_blobs (mask/mask_transform.py:195-323), which the reference runs on the host in the middle of the forward.
//
// Launches (none synchronises the host; every count stays on the device):
//   1. pt_assign: per roidb row (G gt rows, then the rois rows): the gt rows' values from the entry; a proposal's IoU
//                 against every gt row of class > 0 (boxes staged through shared memory), max, first argmax, class
//   2. pt_sample: one CTA of 1024 threads: fg / bg candidate lists in row order, both draws (an exact 8-pass radix
//                 select of the k-th smallest key, the keys recomputed from the positions), the output rows, box
//                 targets, nongt_inds and the counts.  The candidates number R + G, a few thousand: one CTA selects
//                 them in a few microseconds, where the anchor case's multi-kernel passes would cost more in launches.
//   3. pt_mask:   one CTA per mask row: the object of largest IoU with the row's box, its polygons rasterised at M x M
//                 by the rleFrPoly rule (toggles + prefix XOR, below), and the K * M^2 class-specific target row.
//
// The rasteriser is rleFrPoly's edge walk of poly.cuh at h = w = M: each edge's surviving boundary points toggle bits
// of a column-major M x M bitmap in shared memory, and a prefix XOR gives the mask.
#include "common.cuh"
#include "cta.cuh"
#include "poly.cuh"
#include "targets.cuh"

namespace ups {

constexpr int kPtThreads = 256;
constexpr int kPtChunk = 1024;
constexpr int kPtMaxG = UPSNET_RPN_TARGETS_MAX_G;
constexpr int kPtSample = 1024;
constexpr int kPtMaxBatch = 4096;
constexpr int kPtMaxM = 32;          // M * M bits fit one 32-bit word per lane of one warp

enum { kSlotValid = 1 };

struct PtParams {
  const float* rois;                // [R,5]
  const float* gt;                  // [G,4]
  const float* gt_ovl;              // [G] max of gt_overlaps
  const int* gt_maxcls;             // [G] argmax of gt_overlaps
  const int* gt_cls;                // [G] gt_classes
  const int* gt_map;                // [G] box_to_gt_ind_map
  const float* obj_box;             // [O,4]
  const int* obj_poly;              // [O+1]
  const int* poly_vert;             // [P+1]
  const float* verts;               // [V,2]
  int R, G, S, O;
  float im_scale, inv_scale;
  int K, batch, fg_per_image, M;
  float fg_thresh, bg_hi, bg_lo;
  float4 weights;
  unsigned long long seed;
  // workspace
  float* ovl;                       // [S]
  int* cls;                         // [S]
  int* map;                         // [S]
  unsigned char* flags;             // [S]
  int* list[2];                     // [S] fg / bg candidates (slots) in row order
  float4* rowbox;                   // [batch] sampled boxes (unscaled)
  // outputs
  float* rois_out;
  int64_t* labels;
  float *targets, *inside, *outside;
  int64_t* nongt;
  float* mask_rois;
  float* mask;
  unsigned char* has_mask;
  int* counts;
};

__device__ __forceinline__ float4 ld_box(const float* b, int k) {
  return make_float4(__ldg(b + 4 * k), __ldg(b + 4 * k + 1), __ldg(b + 4 * k + 2), __ldg(b + 4 * k + 3));
}

// roidb row `slot`: a gt box, or a proposal rois[r, 1:] * float32(1 / im_scale) (numpy >= 2 keeps float32)
__device__ __forceinline__ float4 slot_box(const PtParams& p, int slot) {
  if (slot < p.G) return ld_box(p.gt, slot);
  const float* r = p.rois + 5 * (size_t)(slot - p.G);
  return make_float4(__fmul_rn(__ldg(r + 1), p.inv_scale), __fmul_rn(__ldg(r + 2), p.inv_scale),
                     __fmul_rn(__ldg(r + 3), p.inv_scale), __fmul_rn(__ldg(r + 4), p.inv_scale));
}

// 1. per roidb row: max overlap, its class and gt row (add_proposals with crowd_thresh = 0)
__global__ void __launch_bounds__(kPtThreads) pt_assign_kernel(const PtParams p) {
  __shared__ float4 sbox[kPtChunk];
  __shared__ float sarea[kPtChunk];
  __shared__ int scls[kPtChunk];
  const int slot = blockIdx.x * kPtThreads + threadIdx.x;
  const bool prop = slot >= p.G && slot < p.S;
  bool valid = false;
  float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
  if (prop) {
    valid = __ldg(p.rois + 5 * (size_t)(slot - p.G)) == 0.f;     // np.where(rois[:, 0] == 0)
    b = slot_box(p, slot);
  }
  const double b_area = area64(b);
  float best = -1.f;
  int arg = -1;
  // only CTAs holding proposals walk the boxes (the condition is uniform over the CTA)
  const bool walk = (blockIdx.x + 1) * kPtThreads > p.G;
  for (int c0 = 0; walk && c0 < p.G; c0 += kPtChunk) {
    const int cn = min(kPtChunk, p.G - c0);
    __syncthreads();
    for (int k = threadIdx.x; k < cn; k += kPtThreads) {
      const float4 q = ld_box(p.gt, c0 + k);
      sbox[k] = q;
      sarea[k] = (float)area64(q);
      scls[k] = __ldg(p.gt_cls + c0 + k);
    }
    __syncthreads();
    if (valid) {
      for (int k = 0; k < cn; ++k) {
        if (scls[k] <= 0) continue;                              // gt_inds: class > 0, crowd included
        const float o = pair_iou(b, b_area, sbox[k], sarea[k]);
        if (o > best) { best = o; arg = c0 + k; }                // strict: the first argmax
      }
    }
  }
  if (slot < p.G) {
    p.ovl[slot] = __ldg(p.gt_ovl + slot);
    p.cls[slot] = __ldg(p.gt_maxcls + slot);
    p.map[slot] = __ldg(p.gt_map + slot);
    p.flags[slot] = kSlotValid;
  } else if (prop) {
    const bool pos = best > 0.f;
    p.ovl[slot] = pos ? best : 0.f;
    p.cls[slot] = pos ? __ldg(p.gt_cls + arg) : 0;
    p.map[slot] = pos ? arg : -1;
    p.flags[slot] = valid ? kSlotValid : 0;
  }
}

// one output row: the roidb row `slot`, fg (label = its class) or bg (label 0)
__device__ void pt_write_row(const PtParams& p, int o, int slot, bool fg, unsigned char* s_nongt) {
  const float4 b = slot_box(p, slot);
  const int label = fg ? p.cls[slot] : 0;
  p.labels[o] = label;
  p.rowbox[o] = b;
  float* r = p.rois_out + 5 * (size_t)o;
  r[0] = 0.f;
  r[1] = __fmul_rn(b.x, p.im_scale); r[2] = __fmul_rn(b.y, p.im_scale);
  r[3] = __fmul_rn(b.z, p.im_scale); r[4] = __fmul_rn(b.w, p.im_scale);
  p.has_mask[o] = label > 0 ? 1 : 0;
  s_nongt[o] = slot >= p.G;         // gt_classes == 0: the proposals (every gt row has a class > 0)
  if (label > 0) {
    int g = p.map[slot];             // gt_inds[box_to_gt_ind_map[keep]], gt_inds = 0..G-1 here
    if (g < 0) g += p.G;
    const float4 t = box_target(b, ld_box(p.gt, g), p.weights);
    const size_t base = (size_t)o * 4 * p.K + 4 * (size_t)label;
    p.targets[base] = t.x; p.targets[base + 1] = t.y; p.targets[base + 2] = t.z; p.targets[base + 3] = t.w;
    for (int c = 0; c < 4; ++c) { p.inside[base + c] = 1.f; p.outside[base + c] = 1.f; }
  }
}

// 2. candidates, draws and the output rows (one CTA)
__global__ void __launch_bounds__(kPtSample) pt_sample_kernel(const PtParams p) {
  __shared__ int warp_sums[kPtSample / 32];
  __shared__ unsigned char s_nongt[kPtMaxBatch];
  int n[2] = {0, 0};
  for (int c0 = 0; c0 < p.S; c0 += kPtSample) {
    const int slot = c0 + threadIdx.x;
    bool fg = false, bg = false;
    if (slot < p.S && (p.flags[slot] & kSlotValid)) {
      const float m = p.ovl[slot];
      fg = m >= p.fg_thresh;
      bg = m < p.bg_hi && m >= p.bg_lo;
    }
    int tf, tb;
    const int ef = cta_scan_excl<kPtSample>((int)fg, warp_sums, &tf);
    const int eb = cta_scan_excl<kPtSample>((int)bg, warp_sums, &tb);
    if (fg) p.list[0][n[0] + ef] = slot;
    if (bg) p.list[1][n[1] + eb] = slot;
    n[0] += tf; n[1] += tb;
  }
  // fg_rois_per_this_image = min(fg_per_image, #fg); bg = min(batch - that, #bg)
  const int take[2] = {min(p.fg_per_image, n[0]), min(p.batch - min(p.fg_per_image, n[0]), n[1])};
  __syncthreads();                  // the candidate lists are complete
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    const int k = take[s], cnt = n[s];
    // the k-th smallest key of the draw, the keys recomputed from the positions
    auto key_at = [&](int i) { return draw_key(p.seed, s, (unsigned long long)i); };
    const unsigned long long kth =
        (k > 0 && k < cnt) ? cta_radix_select<kPtSample, unsigned long long, 64, 8, false>(key_at, cnt, k) : 0ull;
    int base = s ? take[0] : 0;
    for (int c0 = 0; c0 < cnt && k > 0; c0 += kPtSample) {
      const int i = c0 + threadIdx.x;
      const bool sel = i < cnt && (k == cnt || key_at(i) <= kth);
      int tot;
      const int e = cta_scan_excl<kPtSample>((int)sel, warp_sums, &tot);
      if (sel) pt_write_row(p, base + e, p.list[s][i], s == 0, s_nongt);
      base += tot;
    }
  }
  __syncthreads();
  const int nf = take[0], nb = take[1], rows = nf + nb;
  const int nmask = nf > 0 ? nf : (nb > 0 ? 1 : 0);
  int nn = 0;
  for (int c0 = 0; c0 < rows; c0 += kPtSample) {
    const int o = c0 + threadIdx.x;
    const bool f = o < rows && s_nongt[o];
    int tot;
    const int e = cta_scan_excl<kPtSample>((int)f, warp_sums, &tot);
    if (f) p.nongt[nn + e] = o;
    nn += tot;
  }
  // mask_rois: the fg rows, or the first bg row when there is no fg (add_mask_rcnn_blobs' fallback)
  for (int i = threadIdx.x; i < 5 * nmask; i += kPtSample) p.mask_rois[i] = p.rois_out[i];
  if (threadIdx.x == 0) {
    if (nf == 0 && nb > 0) p.has_mask[0] = 1;
    p.counts[0] = nf;
    p.counts[1] = nb;
    p.counts[2] = nmask;
    p.counts[3] = rows == 0;        // the reference raises IndexError (bg_inds[0] of an empty list)
    p.counts[4] = nn;
  }
}

// 3. one mask row: the class-specific K * M^2 target (-1 outside the class slot)
__global__ void __launch_bounds__(kPtThreads) pt_mask_kernel(const PtParams p) {
  __shared__ unsigned int bits[kPtMaxM * kPtMaxM / 32 + 1];
  __shared__ unsigned int acc[kPtMaxM * kPtMaxM / 32];
  __shared__ float s_val[kPtThreads / 32];
  __shared__ int s_idx[kPtThreads / 32];
  const int i = blockIdx.x, M = p.M, MM = M * M, W = (MM + 31) / 32;
  const int label = i < p.counts[2] ? (int)p.labels[i] : 0;
  if (threadIdx.x < 32) acc[threadIdx.x] = 0u;
  if (label > 0) {
    const float4 b = p.rowbox[i];
    const double b_area = area64(b);
    // the object: first argmax of the IoU against the polygons' boxes
    float best = -1.f;
    int arg = 0;
    for (int j = threadIdx.x; j < p.O; j += kPtThreads) {
      const float4 q = ld_box(p.obj_box, j);
      const float o = pair_iou(b, b_area, q, (float)area64(q));
      if (o > best) { best = o; arg = j; }
    }
    for (int off = 16; off; off >>= 1) {
      const float ov = __shfl_down_sync(0xffffffffu, best, off);
      const int oa = __shfl_down_sync(0xffffffffu, arg, off);
      if (ov > best || (ov == best && oa < arg)) { best = ov; arg = oa; }
    }
    if ((threadIdx.x & 31) == 0) { s_val[threadIdx.x >> 5] = best; s_idx[threadIdx.x >> 5] = arg; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < kPtThreads / 32; ++w)
        if (s_val[w] > s_val[0] || (s_val[w] == s_val[0] && s_idx[w] < s_idx[0])) { s_val[0] = s_val[w]; s_idx[0] = s_idx[w]; }
    }
    __syncthreads();
    const int obj = s_idx[0];
    // polys_to_mask_wrt_box's frame, float32: ((p - x1) * M) / max(x2 - x1, 1)
    const float wx = fmaxf(__fsub_rn(b.z, b.x), 1.f), wy = fmaxf(__fsub_rn(b.w, b.y), 1.f), fM = (float)M;
    for (int pg = p.obj_poly[obj]; pg < p.obj_poly[obj + 1]; ++pg) {
      const int v0 = p.poly_vert[pg], k = p.poly_vert[pg + 1] - v0;
      if (threadIdx.x <= W) bits[threadIdx.x] = 0u;
      __syncthreads();
      for (int e = threadIdx.x; e < k; e += kPtThreads) {
        const float* a = p.verts + 2 * (size_t)(v0 + e);
        const float* c = p.verts + 2 * (size_t)(v0 + (e + 1 == k ? 0 : e + 1));
        const int X0 = up5(__fdiv_rn(__fmul_rn(__fsub_rn(a[0], b.x), fM), wx));
        const int Y0 = up5(__fdiv_rn(__fmul_rn(__fsub_rn(a[1], b.y), fM), wy));
        const int X1 = up5(__fdiv_rn(__fmul_rn(__fsub_rn(c[0], b.x), fM), wx));
        const int Y1 = up5(__fdiv_rn(__fmul_rn(__fsub_rn(c[1], b.y), fM), wy));
        edge_toggles(bits, M, M, X0, Y0, X1, Y1);
      }
      __syncthreads();
      if (threadIdx.x < 32) {         // prefix XOR over the column-major bits, OR-ed into the union of the polygons
        const int lane = threadIdx.x;
        const unsigned int w0 = lane < W ? bits[lane] : 0u;
        unsigned int x = w0;
        x ^= x << 1; x ^= x << 2; x ^= x << 4; x ^= x << 8; x ^= x << 16;
        unsigned int par = __popc(w0) & 1u;
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned int y = __shfl_up_sync(0xffffffffu, par, o);
          if (lane >= o) par ^= y;
        }
        const unsigned int carry = par ^ (__popc(w0) & 1u);
        if (lane < W) acc[lane] |= carry ? ~x : x;
      }
      __syncthreads();
    }
  }
  __syncthreads();
  float* row = p.mask + (size_t)i * p.K * MM;
  const int n = p.K * MM;
  for (int j = threadIdx.x; j < n; j += kPtThreads) {
    float v = -1.f;
    const int c = j / MM;
    if (label > 0 && c == label) {
      const int w = j - c * MM, y = w / M, x = w - y * M, a = x * M + y;    // [y][x] out, column-major bits
      v = (float)((acc[a >> 5] >> (a & 31)) & 1u);
    }
    row[j] = v;
  }
}

inline size_t pt_layout(int S, int batch, void* base, PtParams& p) {
  WsCarve c(base);
  p.ovl = c.take<float>(S);
  p.cls = c.take<int>(S);
  p.map = c.take<int>(S);
  p.flags = c.take<unsigned char>(S);
  p.list[0] = c.take<int>(S);
  p.list[1] = c.take<int>(S);
  p.rowbox = c.take<float4>(batch);
  return c.bytes();
}

}  // namespace ups

extern "C" int upsnet_proposal_targets_workspace_bytes(int num_rois, int num_gt, int batch_rois, size_t* bytes) {
  if (!bytes || num_rois < 0 || num_gt <= 0 || batch_rois <= 0) return UPSNET_E_BADARG;
  ups::PtParams p{};
  *bytes = ups::pt_layout(num_rois + num_gt, batch_rois, nullptr, p);
  return 0;
}

extern "C" int upsnet_proposal_targets(
    const float* rois, int R, const float* gt_boxes, const float* gt_max_overlaps, const int* gt_max_classes,
    const int* gt_classes, const int* gt_box_to_gt_ind, int G, const float* obj_boxes, const int* obj_poly_off,
    const int* poly_vert_off, const float* verts, int num_objects, float im_scale, int num_classes, int batch_rois,
    int fg_per_image, float fg_thresh, float bg_thresh_hi, float bg_thresh_lo, float wx, float wy, float ww, float wh,
    int cls_agnostic_bbox_reg, int mask_size, unsigned long long seed, float* rois_out, int64_t* labels,
    float* bbox_targets, float* bbox_inside_weights, float* bbox_outside_weights, int64_t* nongt_inds, float* mask_rois,
    float* mask_int32, unsigned char* roi_has_mask, int* counts, void* workspace, size_t workspace_bytes,
    void* stream) {
  using namespace ups;
  if ((R > 0 && !rois) || !gt_boxes || !gt_max_overlaps || !gt_max_classes || !gt_classes || !gt_box_to_gt_ind ||
      !obj_boxes || !obj_poly_off || !poly_vert_off || !verts || !rois_out || !labels || !bbox_targets ||
      !bbox_inside_weights || !bbox_outside_weights || !nongt_inds || !mask_rois || !mask_int32 || !roi_has_mask ||
      !counts || !workspace)
    return UPSNET_E_BADARG;
  if (R < 0 || G <= 0 || num_objects <= 0 || num_classes <= 0 || batch_rois <= 0 || fg_per_image < 0 ||
      fg_per_image > batch_rois || mask_size <= 0 || !(fg_thresh > 0.f) || !(im_scale > 0.f))
    return UPSNET_E_BADARG;
  if (cls_agnostic_bbox_reg || G > kPtMaxG || mask_size > kPtMaxM || batch_rois > kPtMaxBatch) return UPSNET_E_UNSUPPORTED;
  const int S = R + G;
  PtParams p{};
  if (workspace_bytes < pt_layout(S, batch_rois, workspace, p)) return UPSNET_E_WORKSPACE;
  p.rois = rois; p.gt = gt_boxes; p.gt_ovl = gt_max_overlaps; p.gt_maxcls = gt_max_classes; p.gt_cls = gt_classes;
  p.gt_map = gt_box_to_gt_ind; p.obj_box = obj_boxes; p.obj_poly = obj_poly_off; p.poly_vert = poly_vert_off;
  p.verts = verts;
  p.R = R; p.G = G; p.S = S; p.O = num_objects;
  p.im_scale = im_scale;
  p.inv_scale = 1.0f / im_scale;               // 1. / np.float32 stays float32 (IEEE division on the host)
  p.K = num_classes; p.batch = batch_rois; p.fg_per_image = fg_per_image; p.M = mask_size;
  p.fg_thresh = fg_thresh; p.bg_hi = bg_thresh_hi; p.bg_lo = bg_thresh_lo;
  p.weights = make_float4(wx, wy, ww, wh);
  p.seed = seed;
  p.rois_out = rois_out; p.labels = labels; p.targets = bbox_targets; p.inside = bbox_inside_weights;
  p.outside = bbox_outside_weights; p.nongt = nongt_inds; p.mask_rois = mask_rois; p.mask = mask_int32;
  p.has_mask = roi_has_mask; p.counts = counts;
  const int mcap = fg_per_image > 0 ? fg_per_image : 1;
  const size_t tb = (size_t)batch_rois * 4 * num_classes * 4;
  cudaStream_t st = (cudaStream_t)stream;
  // padding: zero rows, nongt_inds -1 (all bytes 0xff)
  UPS_CUDA(cudaMemsetAsync(rois_out, 0, (size_t)batch_rois * 20, st));
  UPS_CUDA(cudaMemsetAsync(labels, 0, (size_t)batch_rois * 8, st));
  UPS_CUDA(cudaMemsetAsync(bbox_targets, 0, tb, st));
  UPS_CUDA(cudaMemsetAsync(bbox_inside_weights, 0, tb, st));
  UPS_CUDA(cudaMemsetAsync(bbox_outside_weights, 0, tb, st));
  UPS_CUDA(cudaMemsetAsync(nongt_inds, 0xff, (size_t)batch_rois * 8, st));
  UPS_CUDA(cudaMemsetAsync(roi_has_mask, 0, (size_t)batch_rois, st));
  UPS_CUDA(cudaMemsetAsync(mask_rois, 0, (size_t)mcap * 20, st));
  pt_assign_kernel<<<(S + kPtThreads - 1) / kPtThreads, kPtThreads, 0, st>>>(p);
  UPS_CHECK_LAUNCH();
  pt_sample_kernel<<<1, kPtSample, 0, st>>>(p);
  UPS_CHECK_LAUNCH();
  pt_mask_kernel<<<mcap, kPtThreads, 0, st>>>(p);
  UPS_CHECK_LAUNCH();
  return 0;
}
