// cocoeval.cu -- COCO box / mask AP (pycocotools COCOeval with its default Params, iouType 'bbox' or 'segm'), device
// resident (evaluation half of SURVEY section 8f row f4):
//
//  * upsnet_cocoeval_image: COCOeval.evaluate() for one image -- _prepare (ignore = iscrowd), computeIoU (maskApi.c bbIou /
//    rleIou) and evaluateImg for the 10 IoU thresholds x 4 area ranges at maxDet 100.  One CTA per category: it gathers
//    the category's detections (stable rank by descending score, the first 100 kept) and ground truths, computes their
//    IoU matrix in shared memory, and runs the 40 greedy matchings, one thread each.  It writes one record per kept
//    detection (score, category, image slot, rank, matched / ignored bits of the 40 (threshold, area) pairs) and adds the
//    non-ignored ground-truth counts to npig [K][4].  Masks are never decoded: run lengths are prefix-summed into run
//    boundaries, and the intersection of two masks walks the detection's runs of ones with a binary search into the
//    ground truth's boundaries.
//  * upsnet_cocoeval_accumulate: COCOeval.accumulate() over every record -- one stable radix sort of all records by
//    (category, -score, image-id rank, rank in image), then per (category, area, maxDet) one warp per IoU threshold
//    that forms the cumulative tp / fp counts, recall, precision, its envelope and the 101 recall-threshold lookups.
// Every product and sum that reaches a result is spelled with an explicit round-to-nearest intrinsic, so no FMA
// contraction can make the device differ from the numpy oracle.
#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"

namespace ups {

constexpr int kCocoThreads = 256;
constexpr int kCocoKeep = 100;                                   // Params.maxDets[-1]
constexpr int kCocoT = 10, kCocoA = 4, kCocoM = 3, kCocoR = 101;
constexpr int kCocoMaxDet = UPSNET_COCOEVAL_MAX_DET;
constexpr int kCocoMaxGt = UPSNET_COCOEVAL_MAX_GT;
constexpr int kCocoMaxGtCat = UPSNET_COCOEVAL_MAX_GT_CAT;
static_assert(kCocoT * kCocoA <= 64, "matched / ignored bits of one record fit in 64 bits");

// Params: iouThrs = np.linspace(.5, .95, 10), recThrs = np.linspace(0, 1, 101) -- numpy's linspace is
// start + i * ((stop - start) / (num - 1)) with the last entry set to stop.
__device__ __forceinline__ double coco_iou_thr(int t) {
  return t == kCocoT - 1 ? 0.95 : __dadd_rn(__dmul_rn((double)t, (0.95 - 0.5) / 9.0), 0.5);
}
__device__ __forceinline__ double coco_rec_thr(int r) { return r == kCocoR - 1 ? 1.0 : __dmul_rn((double)r, 1.0 / 100.0); }
// areaRng [[0, 1e5**2], [0, 32**2], [32**2, 96**2], [96**2, 1e5**2]], both ends inclusive
__device__ __forceinline__ bool coco_out_of_range(double area, int a) {
  const double lo = a == 2 ? 1024.0 : (a == 3 ? 9216.0 : 0.0);
  const double hi = a == 1 ? 1024.0 : (a == 2 ? 9216.0 : 1e10);
  return area < lo || area > hi;
}

struct CocoSmem {
  double iou[kCocoKeep * kCocoMaxGtCat];          // [rank][gt of the category]
  double gbox[4][kCocoMaxGtCat];
  double garea[kCocoMaxGtCat];                    // the annotation's `area` (the area-range test)
  double dbox[4][kCocoKeep];                      // x, y, w, h as the reference's xyxy_to_xywh makes them (float64)
  double darea[kCocoKeep];                        // w * h (bbox) or the RLE pixel count (segm)
  unsigned long long mbits[kCocoKeep], ibits[kCocoKeep];
  int dlist[kCocoMaxDet];                         // detections of this category, input order
  int keep[kCocoKeep];                            // detection of rank r
  int glist[kCocoMaxGtCat];                       // ground-truth rows of this category, table order
  unsigned dfirst[kCocoKeep], dlast[kCocoKeep], gfirst[kCocoMaxGtCat], glast[kCocoMaxGtCat], grle_area[kCocoMaxGtCat];
  unsigned short gord[kCocoA][kCocoMaxGtCat];     // gt order after the stable sort by _ignore
  unsigned char gcrowd[kCocoMaxGtCat], gig[kCocoA][kCocoMaxGtCat];
  unsigned char gtm[kCocoT * kCocoA][kCocoMaxGtCat];
  int warp_n[kCocoThreads / 32];
  int nd, ng, rec_base, err;
};
static_assert(sizeof(CocoSmem) <= 227 * 1024, "one category's state fits in shared memory");

// Appends the indices i < n with pred(i) to out[] in ascending order (a block-wide ballot scan); returns the count
// (every thread gets it).  `cap` bounds the writes; the returned count is not clamped.
template <typename Pred>
__device__ int block_compact(int n, int* out, int cap, int* warp_n, Pred pred) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int total = 0;
  for (int base = 0; base < n; base += kCocoThreads) {
    const int i = base + threadIdx.x;
    const bool f = i < n && pred(i);
    const unsigned bal = __ballot_sync(0xffffffffu, f);
    if (lane == 0) warp_n[warp] = __popc(bal);
    __syncthreads();
    int off = total;
    for (int w = 0; w < warp; ++w) off += warp_n[w];
    off += __popc(bal & ((1u << lane) - 1u));
    if (f && off < cap) out[off] = i;
    int sum = 0;
    for (int w = 0; w < kCocoThreads / 32; ++w) sum += warp_n[w];
    total += sum;
    __syncthreads();
  }
  return total;
}

// Run boundaries of one COCO RLE (warp-cooperative): bnd[j] = cnt[0] + ... + cnt[j], the end of run j; runs of odd j are
// ones.  Returns the pixel total; *area = pixels in runs of ones; [*first, *last) covers every one (empty when no ones).
__device__ unsigned rle_bounds(const unsigned* __restrict__ cnt, int len, unsigned* __restrict__ bnd, unsigned* area,
                               unsigned* first, unsigned* last) {
  const int lane = threadIdx.x & 31;
  unsigned carry = 0, ones = 0;
  for (int base = 0; base < len; base += 32) {
    const int j = base + lane;
    const unsigned c = j < len ? cnt[j] : 0u;
    unsigned s = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned v = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += v;
    }
    if (j < len) bnd[j] = carry + s;
    if (j & 1) ones += c;
    carry += __shfl_sync(0xffffffffu, s, 31);
  }
  ones = __reduce_add_sync(0xffffffffu, ones);
  __syncwarp();
  if (lane == 0) {
    *area = ones;
    const int lo = len >= 2 ? ((len & 1) ? len - 2 : len - 1) : -1;     // last run of ones
    *first = lo >= 0 ? bnd[0] : 0u;
    *last = lo >= 0 ? bnd[lo] : 0u;
  }
  return carry;
}

// Pixels shared by two masks given by run boundaries (warp-cooperative): each lane takes runs of ones of the detection
// and finds the overlapping ground-truth runs by binary search.
__device__ unsigned rle_intersection(const unsigned* __restrict__ bd, int nd, const unsigned* __restrict__ bg, int ng) {
  const int lane = threadIdx.x & 31;
  unsigned inter = 0;
  for (int j = 2 * lane + 1; j < nd; j += 64) {
    const unsigned s = bd[j - 1], e = bd[j];
    if (s >= e) continue;
    int lo = 0, hi = ng;                                          // first q with bg[q] > s: the gt run holding pixel s
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (bg[mid] <= s) lo = mid + 1; else hi = mid; }
    for (int q = lo; q < ng; ++q) {
      const unsigned gs = q ? bg[q - 1] : 0u;
      if (gs >= e) break;
      if (q & 1) inter += min(e, bg[q]) - max(s, gs);
    }
  }
  return __reduce_add_sync(0xffffffffu, inter);
}

struct CocoImageArgs {
  const float* boxes; const float* scores; const long long* cls; int n; const int* n_dev;
  const unsigned* counts; int cap; const int* run_len; int H, W;
  const double* gt; int G; const unsigned* gt_counts; const long long* gt_off;
  int K; const int* cls_to_k; int image;
  upsnet_coco_record* rec; int rec_cap; int* n_rec; long long* npig; int* err;
  unsigned* det_bnd; unsigned* gt_bnd;                            // workspace: [n][cap] and [gt_off[G]]
  int segm;
};

__global__ void __launch_bounds__(kCocoThreads)
coco_image_kernel(const __grid_constant__ CocoImageArgs p) {
  extern __shared__ __align__(16) unsigned char coco_smem[];
  CocoSmem& s = *reinterpret_cast<CocoSmem*>(coco_smem);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, c = blockIdx.x;
  const int n = p.n_dev ? min(*p.n_dev, p.n) : p.n;
  if (n > kCocoMaxDet || n < 0) { if (c == 0 && tid == 0) atomicOr(p.err, UPSNET_COCOEVAL_E_DET_COUNT); return; }
  if (p.G > kCocoMaxGt) { if (c == 0 && tid == 0) atomicOr(p.err, UPSNET_COCOEVAL_E_GT_COUNT); return; }
  if (tid == 0) s.err = 0;
  __syncthreads();
  const double* g_cat = p.gt; const double* g_crowd = p.gt + p.G; const double* g_area = p.gt + 2 * p.G;
  const int K = p.K;
  // detections and ground truths of category c, in input order
  const int nd = block_compact(n, s.dlist, kCocoMaxDet, s.warp_n, [&](int d) {
    const long long k = p.cls[d];
    if (k < 1 || k > K) { if (c == 0) atomicOr(&s.err, UPSNET_COCOEVAL_E_CLASS); return false; }
    return p.cls_to_k[k] == c;
  });
  const int ng = block_compact(p.G, s.glist, kCocoMaxGtCat, s.warp_n, [&](int g) { return (int)g_cat[g] == c; });
  if (ng > kCocoMaxGtCat) {
    if (tid == 0) atomicOr(p.err, UPSNET_COCOEVAL_E_GT_CAT | s.err);
    return;
  }
  if (nd == 0 && ng == 0) { if (tid == 0 && s.err) atomicOr(p.err, s.err); return; }
  const int nk = min(nd, kCocoKeep);
  // stable rank by descending score (np.argsort(-score, kind='mergesort')), ties in input order
  for (int i = tid; i < nd; i += kCocoThreads) {
    const float si = p.scores[s.dlist[i]];
    int r = 0;
    for (int j = 0; j < nd; ++j) {
      const float sj = p.scores[s.dlist[j]];
      r += (sj > si) || (sj == si && j < i);
    }
    if (r < kCocoKeep) s.keep[r] = s.dlist[i];
  }
  for (int g = tid; g < ng; g += kCocoThreads) {
    const int row = s.glist[g];
    s.gcrowd[g] = g_crowd[row] != 0.0;
    s.garea[g] = g_area[row];
    for (int q = 0; q < 4; ++q) s.gbox[q][g] = p.gt[(3 + q) * p.G + row];
    if (p.segm && ((int)p.gt[7 * p.G + row] != p.H || (int)p.gt[8 * p.G + row] != p.W)) atomicOr(&s.err, UPSNET_COCOEVAL_E_RLE_SIZE);
  }
  __syncthreads();
  for (int r = tid; r < nk; r += kCocoThreads) {
    const int d = s.keep[r];
    s.mbits[r] = 0ull; s.ibits[r] = 0ull;
    // dets.astype(float); xyxy_to_xywh: w = x2 - x1 + 1 in float64
    const double x1 = p.boxes[4 * d], y1 = p.boxes[4 * d + 1], x2 = p.boxes[4 * d + 2], y2 = p.boxes[4 * d + 3];
    s.dbox[0][r] = x1; s.dbox[1][r] = y1;
    s.dbox[2][r] = __dadd_rn(__dsub_rn(x2, x1), 1.0);
    s.dbox[3][r] = __dadd_rn(__dsub_rn(y2, y1), 1.0);
    if (!p.segm) s.darea[r] = __dmul_rn(s.dbox[2][r], s.dbox[3][r]);            // loadRes: bb[2] * bb[3]
  }
  // ground-truth order per area range: stable sort by _ignore (np.argsort(gtIg, kind='mergesort'))
  for (int a = warp; a < kCocoA; a += kCocoThreads / 32) {
    int base = 0;
    for (int pass = 0; pass < 2; ++pass)
      for (int g0 = 0; g0 < ng; g0 += 32) {
        const int g = g0 + lane;
        const bool ig = g < ng && (s.gcrowd[g] || coco_out_of_range(s.garea[g], a));
        if (g < ng) s.gig[a][g] = ig;
        const bool take = g < ng && ig == (pass == 1);
        const unsigned bal = __ballot_sync(0xffffffffu, take);
        if (take) s.gord[a][base + __popc(bal & ((1u << lane) - 1u))] = (unsigned short)g;
        base += __popc(bal);
      }
  }
  for (int i = tid; i < kCocoT * kCocoA * ng; i += kCocoThreads) s.gtm[i / ng][i % ng] = 0;
  if (p.segm) {
    // run boundaries of the kept detections and of the category's ground truths, one warp per RLE
    const long long HW = (long long)p.H * p.W;
    for (int r = warp; r < nk; r += kCocoThreads / 32) {
      const int d = s.keep[r], len = p.run_len[d];
      if (len > p.cap || len < 0) {                               // im_post_rle overflowed its buffer: runs unknown
        if (lane == 0) { atomicOr(&s.err, UPSNET_COCOEVAL_E_RLE_SIZE); s.darea[r] = 0.0; s.dfirst[r] = s.dlast[r] = 0u; }
        continue;
      }
      unsigned area;
      const unsigned tot = rle_bounds(p.counts + (size_t)d * p.cap, len, p.det_bnd + (size_t)d * p.cap, &area, &s.dfirst[r], &s.dlast[r]);
      if (lane == 0) {
        s.darea[r] = (double)area;                                // maskUtils.area
        if (HW && (long long)tot != HW) atomicOr(&s.err, UPSNET_COCOEVAL_E_RLE_SIZE);
      }
    }
    for (int g = warp; g < ng; g += kCocoThreads / 32) {
      const int row = s.glist[g];
      const long long o = p.gt_off[row];
      const unsigned tot = rle_bounds(p.gt_counts + o, (int)(p.gt_off[row + 1] - o), p.gt_bnd + o, &s.grle_area[g], &s.gfirst[g], &s.glast[g]);
      if (lane == 0 && (long long)tot != HW) atomicOr(&s.err, UPSNET_COCOEVAL_E_RLE_SIZE);
    }
  }
  __syncthreads();
  // IoU matrix [rank][gt]
  if (p.segm) {
    for (int i = warp; i < nk * ng; i += kCocoThreads / 32) {
      const int r = i / ng, g = i % ng;
      double v = 0.0;
      if (s.dfirst[r] < s.glast[g] && s.gfirst[g] < s.dlast[r]) {         // disjoint spans of ones: provably 0
        const int d = s.keep[r], row = s.glist[g];
        const long long o = p.gt_off[row];
        const unsigned inter = rle_intersection(p.det_bnd + (size_t)d * p.cap, p.run_len[d], p.gt_bnd + o,
                                                (int)(p.gt_off[row + 1] - o));
        // rleIou: integer intersection and union (or the detection's area against a crowd region), one division
        const unsigned da = (unsigned)s.darea[r];
        const unsigned u = s.gcrowd[g] ? da : da + s.grle_area[g] - inter;
        if (inter) v = __ddiv_rn((double)inter, (double)u);
      }
      if (lane == 0) s.iou[r * ng + g] = v;
    }
  } else {
    for (int i = tid; i < nk * ng; i += kCocoThreads) {
      const int r = i / ng, g = i % ng;
      // bbIou: w = fmin(D[2]+D[0], G[2]+G[0]) - fmax(D[0], G[0]), u = crowd ? da : da + ga - i
      const double dx = s.dbox[0][r], dy = s.dbox[1][r], dw = s.dbox[2][r], dh = s.dbox[3][r];
      const double gx = s.gbox[0][g], gy = s.gbox[1][g], gw = s.gbox[2][g], gh = s.gbox[3][g];
      double v = 0.0;
      const double w = __dsub_rn(fmin(__dadd_rn(dw, dx), __dadd_rn(gw, gx)), fmax(dx, gx));
      if (w > 0) {
        const double h = __dsub_rn(fmin(__dadd_rn(dh, dy), __dadd_rn(gh, gy)), fmax(dy, gy));
        if (h > 0) {
          const double in = __dmul_rn(w, h), da = __dmul_rn(dw, dh), ga = __dmul_rn(gw, gh);
          const double u = s.gcrowd[g] ? da : __dsub_rn(__dadd_rn(da, ga), in);
          v = __ddiv_rn(in, u);
        }
      }
      s.iou[r * ng + g] = v;
    }
  }
  __syncthreads();
  // evaluateImg: one greedy matching per (threshold, area range)
  if (tid < kCocoT * kCocoA) {
    const int t = tid % kCocoT, a = tid / kCocoT;
    unsigned char* gtm = s.gtm[tid];
    const unsigned char* ig = s.gig[a];
    const unsigned short* ord = s.gord[a];
    const double thr = fmin(coco_iou_thr(t), 1.0 - 1e-10);
    const unsigned long long bit = 1ull << tid;
    for (int r = 0; r < nk; ++r) {
      double best = thr;
      int m = -1;
      for (int j = 0; j < ng; ++j) {
        const int g = ord[j];
        if (gtm[g] && !s.gcrowd[g]) continue;                   // already matched, not a crowd
        if (m > -1 && !ig[m] && ig[g]) break;                   // matched a regular gt, the ignored block starts
        const double v = s.iou[r * ng + g];
        if (v < best) continue;
        best = v;
        m = g;
      }
      if (m >= 0) {
        gtm[m] = 1;
        atomicOr(&s.mbits[r], bit);
        if (ig[m]) atomicOr(&s.ibits[r], bit);
      } else if (coco_out_of_range(s.darea[r], a)) {
        atomicOr(&s.ibits[r], bit);
      }
    }
  }
  if (tid < kCocoA) {
    long long np_ = 0;
    for (int g = 0; g < ng; ++g) np_ += !s.gig[tid][g];
    if (np_) atomicAdd(reinterpret_cast<unsigned long long*>(p.npig + (size_t)c * kCocoA + tid), (unsigned long long)np_);
  }
  if (tid == 0) s.rec_base = nk ? atomicAdd(p.n_rec, nk) : 0;
  __syncthreads();
  if (s.rec_base + nk > p.rec_cap) {
    if (tid == 0) atomicOr(&s.err, UPSNET_COCOEVAL_E_RECORDS);
  } else {
    for (int r = tid; r < nk; r += kCocoThreads) {
      upsnet_coco_record rec;
      rec.score = p.scores[s.keep[r]];
      rec.category = c;
      rec.image = p.image;
      rec.rank = r;
      rec.matched = s.mbits[r];
      rec.ignored = s.ibits[r];
      p.rec[s.rec_base + r] = rec;
    }
  }
  __syncthreads();
  if (tid == 0 && s.err) atomicOr(p.err, s.err);
}

// ---- accumulate ----

__device__ __forceinline__ unsigned long long coco_sort_key(const upsnet_coco_record& r, const int* image_rank) {
  unsigned u = __float_as_uint(r.score + 0.0f);                 // -0 -> +0: the two compare equal in numpy
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);               // ascending float order as unsigned
  return ((unsigned long long)(unsigned)r.category << 56) | ((unsigned long long)(~u) << 24) |
         ((unsigned long long)(unsigned)image_rank[r.image] << 7) | (unsigned long long)(unsigned)r.rank;
}

__global__ void coco_keys_kernel(const upsnet_coco_record* __restrict__ rec, int N, const int* __restrict__ image_rank,
                                 unsigned long long* __restrict__ keys, int* __restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) { keys[i] = coco_sort_key(rec[i], image_rank); vals[i] = i; }
}

__device__ int lower_bound_u64(const unsigned long long* a, int n, unsigned long long v) {
  int lo = 0, hi = n;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[mid] < v) lo = mid + 1; else hi = mid; }
  return lo;
}

// One block per (category, area, maxDet), one warp per IoU threshold.  Pass 1 counts tp / fp / detections; pass 2 walks
// the records backwards so that each one knows its cumulative counts and the envelope (suffix max) of the precision
// from it to the end, and writes the recall thresholds it is the searchsorted(rc, recThrs, 'left') answer for.
__global__ void __launch_bounds__(32 * kCocoT)
coco_accumulate_kernel(const upsnet_coco_record* __restrict__ rec, const unsigned long long* __restrict__ keys,
                       const int* __restrict__ order, int N, const long long* __restrict__ npig, int K,
                       double* __restrict__ precision, double* __restrict__ recall, double* __restrict__ scores) {
  const int k = blockIdx.x, a = blockIdx.y, m = blockIdx.z, t = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int max_det = m == 0 ? 1 : (m == 1 ? 10 : 100);
  const unsigned long long bit = 1ull << (a * kCocoT + t);
  const long long np_ = npig[(size_t)k * kCocoA + a];
  auto at = [&](int r) { return ((((size_t)t * kCocoR + r) * K + k) * kCocoA + a) * kCocoM + m; };
  const size_t rec_at = (((size_t)t * K + k) * kCocoA + a) * kCocoM + m;
  for (int r = lane; r < kCocoR; r += 32) { precision[at(r)] = np_ ? 0.0 : -1.0; scores[at(r)] = np_ ? 0.0 : -1.0; }
  if (!np_) { if (lane == 0) recall[rec_at] = -1.0; return; }
  __syncwarp();
  const int lo = lower_bound_u64(keys, N, (unsigned long long)k << 56);
  const int hi = k + 1 < 256 ? lower_bound_u64(keys, N, (unsigned long long)(k + 1) << 56) : N;
  const double npd = (double)np_, eps = 2.220446049250313e-16;  // np.spacing(1)
  int tp_tot = 0, fp_tot = 0, nd_tot = 0;
  for (int j = lo + lane; j < hi; j += 32) {
    const upsnet_coco_record& r = rec[order[j]];
    if (r.rank >= max_det) continue;
    const bool mt = r.matched & bit, ig = r.ignored & bit;
    nd_tot += 1; tp_tot += mt && !ig; fp_tot += !mt && !ig;
  }
  tp_tot = __reduce_add_sync(0xffffffffu, tp_tot);
  fp_tot = __reduce_add_sync(0xffffffffu, fp_tot);
  nd_tot = __reduce_add_sync(0xffffffffu, nd_tot);
  if (lane == 0) recall[rec_at] = nd_tot ? __ddiv_rn((double)tp_tot, npd) : 0.0;
  int tp_rem = tp_tot, fp_rem = fp_tot, nd_rem = nd_tot;          // counts up to and including the chunk's last record
  double env = 0.0;                                               // max precision after the chunk (precision >= 0)
  for (int end = hi; end > lo; end -= 32) {
    const int j = end - 32 + lane;
    bool valid = false, tpi = false, fpi = false;
    float sc = 0.0f;
    if (j >= lo) {
      const upsnet_coco_record& r = rec[order[j]];
      valid = r.rank < max_det;
      const bool mt = r.matched & bit, ig = r.ignored & bit;
      tpi = valid && mt && !ig; fpi = valid && !mt && !ig; sc = r.score;
    }
    // suffix sums over lanes above this one (later records of the chunk)
    int tp_after = tpi, fp_after = fpi, nd_after = valid;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int a1 = __shfl_down_sync(0xffffffffu, tp_after, o), b1 = __shfl_down_sync(0xffffffffu, fp_after, o),
                c1 = __shfl_down_sync(0xffffffffu, nd_after, o);
      if (lane + o < 32) { tp_after += a1; fp_after += b1; nd_after += c1; }
    }
    const int tp_i = tp_rem - (tp_after - tpi), fp_i = fp_rem - (fp_after - fpi), nd_i = nd_rem - (nd_after - valid);
    double pr = valid ? __ddiv_rn((double)tp_i, __dadd_rn(__dadd_rn((double)fp_i, (double)tp_i), eps)) : 0.0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double v = __shfl_down_sync(0xffffffffu, pr, o);
      if (lane + o < 32) pr = fmax(pr, v);
    }
    pr = fmax(pr, env);                                           // the envelope at this record
    if (valid) {
      const double rc = __ddiv_rn((double)tp_i, npd);
      const double rc_prev = __ddiv_rn((double)(tp_i - tpi), npd);
      const bool first = nd_i == 1;
      if (first || tpi) {
        for (int r = 0; r < kCocoR; ++r) {
          const double thr = coco_rec_thr(r);
          if (thr > rc) break;
          if (first || thr > rc_prev) { precision[at(r)] = pr; scores[at(r)] = (double)sc; }
        }
      }
    }
    env = __shfl_sync(0xffffffffu, pr, 0);
    tp_rem -= __shfl_sync(0xffffffffu, tp_after, 0);
    fp_rem -= __shfl_sync(0xffffffffu, fp_after, 0);
    nd_rem -= __shfl_sync(0xffffffffu, nd_after, 0);
  }
}

}  // namespace ups

extern "C" int upsnet_cocoeval_workspace_bytes(int n, int cap, long long gt_counts_total, size_t* bytes) {
  if (!bytes || n < 0 || cap < 0 || gt_counts_total < 0) return UPSNET_E_BADARG;
  *bytes = ups::align_up(sizeof(unsigned) * (size_t)n * cap, 256) + sizeof(unsigned) * (size_t)gt_counts_total;
  return 0;
}

extern "C" int upsnet_cocoeval_image(int segm, const float* boxes, const float* scores, const int64_t* cls_inds, int n,
                                     const int* n_dev, const uint32_t* counts, int cap, const int* run_len, int H, int W,
                                     const double* gt_table, int num_gt, const uint32_t* gt_counts, const int64_t* gt_offsets,
                                     int num_categories, const int* class_to_k, int image_slot, upsnet_coco_record* records,
                                     int record_cap, int* n_records, long long* npig, int* err, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  using namespace ups;
  if (n < 0 || num_gt < 0 || image_slot < 0 || record_cap < 0) return UPSNET_E_BADARG;
  if (num_categories < 1 || num_categories > UPSNET_COCOEVAL_MAX_CATEGORIES) return UPSNET_E_BADARG;
  if (!class_to_k || !records || !n_records || !npig || !err) return UPSNET_E_BADARG;
  if (n > 0 && (!boxes || !scores || !cls_inds)) return UPSNET_E_BADARG;
  if (num_gt > 0 && num_gt <= kCocoMaxGt && !gt_table) return UPSNET_E_BADARG;
  if (segm && (H < 0 || W < 0 || (n > 0 && (!counts || !run_len || cap <= 0)) ||
               (num_gt > 0 && num_gt <= kCocoMaxGt && (!gt_counts || !gt_offsets))))
    return UPSNET_E_BADARG;
  CocoImageArgs p{boxes, scores, (const long long*)cls_inds, n, n_dev, counts, cap, run_len, H, W,
                  gt_table, num_gt, gt_counts, (const long long*)gt_offsets, num_categories, class_to_k, image_slot,
                  records, record_cap, n_records, npig, err, nullptr, nullptr, segm ? 1 : 0};
  if (segm) {
    // gt_offsets lives on the device: the caller sizes the workspace with the total it staged from the host
    const size_t need = align_up(sizeof(unsigned) * (size_t)n * cap, 256);
    if (!workspace || workspace_bytes < need) return UPSNET_E_WORKSPACE;
    p.det_bnd = (unsigned*)workspace;
    p.gt_bnd = (unsigned*)((char*)workspace + need);
  }
  static PerDeviceOnce configured;
  if (configured.need())
    UPS_CUDA(cudaFuncSetAttribute(coco_image_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CocoSmem)));
  coco_image_kernel<<<num_categories, kCocoThreads, sizeof(CocoSmem), (cudaStream_t)stream>>>(p);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_cocoeval_accumulate_workspace_bytes(int n_records, size_t* bytes) {
  if (!bytes || n_records < 0) return UPSNET_E_BADARG;
  size_t cub_bytes = 0;
  UPS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                           (const int*)nullptr, (int*)nullptr, n_records));
  const size_t n = (size_t)n_records;
  *bytes = 2 * ups::align_up(8 * n, 256) + 2 * ups::align_up(4 * n, 256) + cub_bytes;
  return 0;
}

extern "C" int upsnet_cocoeval_accumulate(const upsnet_coco_record* records, int n_records, const int* image_rank,
                                          const long long* npig, int num_categories, double* precision, double* recall,
                                          double* scores, void* workspace, size_t workspace_bytes, void* stream) {
  using namespace ups;
  if (n_records < 0 || num_categories < 1 || num_categories > UPSNET_COCOEVAL_MAX_CATEGORIES) return UPSNET_E_BADARG;
  if (!npig || !precision || !recall || !scores || (n_records > 0 && (!records || !image_rank))) return UPSNET_E_BADARG;
  size_t need = 0;
  const int rc = upsnet_cocoeval_accumulate_workspace_bytes(n_records, &need);
  if (rc) return rc;
  if (!workspace || workspace_bytes < need) return UPSNET_E_WORKSPACE;
  const size_t n = (size_t)n_records;
  char* w = (char*)workspace;
  unsigned long long* keys_in = (unsigned long long*)w;       w += align_up(8 * n, 256);
  unsigned long long* keys_out = (unsigned long long*)w;      w += align_up(8 * n, 256);
  int* vals_in = (int*)w;                                     w += align_up(4 * n, 256);
  int* vals_out = (int*)w;                                    w += align_up(4 * n, 256);
  size_t cub_bytes = need - (size_t)(w - (char*)workspace);
  cudaStream_t st = (cudaStream_t)stream;
  if (n_records > 0) {
    coco_keys_kernel<<<ceil_div(n_records, 256), 256, 0, st>>>(records, n_records, image_rank, keys_in, vals_in);
    UPS_CHECK_LAUNCH();
    UPS_CUDA(cub::DeviceRadixSort::SortPairs(w, cub_bytes, keys_in, keys_out, vals_in, vals_out, n_records, 0, 64, st));
  }
  coco_accumulate_kernel<<<dim3(num_categories, kCocoA, kCocoM), 32 * kCocoT, 0, st>>>(
      records, keys_out, vals_out, n_records, npig, num_categories, precision, recall, scores);
  UPS_CHECK_LAUNCH();
  return 0;
}
