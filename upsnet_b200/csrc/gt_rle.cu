// gt_rle.cu -- COCO.annToRLE of one image's ground truths (pycocotools maskUtils.merge(maskUtils.frPyObjects(segm, h,
// w))) on the device: every polygon rasterised by maskApi.c rleFrPoly at the image's h x w, the polygons of one
// annotation united as rleMerge(intersect = 0) does, and the union run-length encoded; host run lengths (crowd RLE dicts)
// copied through.  The output is the (gt_counts, gt_offsets) pair upsnet_cocoeval_image reads.
//
// The canvas is cut into bands of kGrBand pixels of the column-major order, and one CTA owns one (band, annotation):
//   * a polygon's value at the pixel before the band is the parity of its toggles below the band start.  Every column
//     n <= ceil(p0 / h) - 2 toggles below it whatever its row, so those are only counted; the few columns at the band
//     and just before it are walked.  The union's value there is the OR of those parities: the band's incoming bit.
//   * an edge's walked columns are spread over the CTA's threads (an exclusive scan of the per-edge column counts, then
//     one thread per (edge, column)), so a long edge is not walked serially by one thread.  Toggles are atomic XORs
//     into a shared-memory bitmap: order-free, so the result does not depend on the schedule.
//   * prefix XOR of each polygon's bitmap, from its incoming parity, OR-ed into the union bitmap; the boundaries of the
//     union (bit i != bit i - 1, the incoming bit before the first) are the run ends.
// Launches (none synchronises the host):
//   1. gt_rle_band_kernel<false>: per (band, annotation) the boundary count and the last boundary.
//   2. gt_rle_scan_kernel: one CTA: per annotation the runs (boundaries + 1, or the host run count), gt_offsets by an
//      exclusive scan, each band's first run index and the boundary before it, the last run of each annotation, and the
//      capacity check (over it: the error flag, every offset 0, nothing written).
//   3. gt_rle_band_kernel<true>: the same rasterisation again, each boundary writing the run it ends; the host runs
//      copied.  Rasterising twice costs less than keeping every band's bitmap in global memory between launches.
// The canonical form: a mask's runs are the differences of its boundaries with 0 before the first and h * w after the
// last, so the first run counts zeros and may be 0 and every later run is > 0 -- what rleFrPoly returns for one polygon
// and rleMerge for several.
#include "common.cuh"
#include "cta.cuh"
#include "poly.cuh"

namespace ups {

constexpr int kGrThreads = 256;
constexpr int kGrWords = 2048;                       // one band's bitmap
constexpr int kGrBand = 32 * kGrWords;               // pixels per band
constexpr int kGrPer = kGrWords / kGrThreads;        // words each thread owns in the prefix XOR and the boundary count
constexpr int kGrScanThreads = 1024;

struct GtRleArgs {
  int h, w, G, nb;
  const int* ann_poly;          // [G+1] polygons of annotation g: [ann_poly[g], ann_poly[g+1]); none: a host RLE
  const int* poly_vert;         // [P+1]
  const double* verts;          // [V,2]
  const long long* src_off;     // [G+1]
  const unsigned* src_counts;
  unsigned* counts;
  long long cap;
  long long* offsets;           // [G+1]
  int* err;
  // workspace, [G][nb] per band
  int* band_n;                  // boundaries in the band
  int* band_last;               // its last boundary (pixel index), -1 when none
  int* band_prev;               // the annotation's last boundary before the band, 0 when none
  long long* band_base;         // index in counts of the run the band's first boundary ends
  int* ann_last;                // [G] the annotation's last boundary, 0 when none
  int* ok;                      // the runs fit in cap
};

// The largest v over the threads below this one in thread order (-1 when there is none).  warp_v is Threads / 32 ints
// of shared memory, free again on return.
template <int Threads>
__device__ __forceinline__ int cta_max_excl(int v, int* warp_v) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x = max(x, y);
  }
  const int below = __shfl_up_sync(0xffffffffu, x, 1);
  if (lane == 31) warp_v[wid] = x;
  __syncthreads();
  int r = lane ? below : -1;
  for (int k = 0; k < wid; ++k) r = max(r, warp_v[k]);
  __syncthreads();
  return r;
}

// The boundaries of the union in word i of the band: bit j set when pixel p0 + 32 i + j differs from the pixel before
__device__ __forceinline__ unsigned band_edges(const unsigned* acc, int i, bool inc, int nbits) {
  const unsigned m = acc[i];
  const unsigned before = i ? acc[i - 1] >> 31 : (unsigned)inc;
  unsigned t = m ^ ((m << 1) | before);
  const int valid = nbits - 32 * i;
  if (valid < 32) t &= valid > 0 ? (1u << valid) - 1u : 0u;
  return t;
}

template <bool Emit>
__global__ void __launch_bounds__(kGrThreads) gt_rle_band_kernel(const GtRleArgs p) {
  __shared__ unsigned bits[kGrWords];               // one polygon's toggles
  __shared__ unsigned acc[kGrWords];                // the union of the polygons so far
  __shared__ PolyEdge s_edge[kGrThreads];
  __shared__ int s_start[kGrThreads];
  __shared__ int warp_i[kGrThreads / 32];
  const int tid = threadIdx.x, b = blockIdx.x, g = blockIdx.y, h = p.h;
  if (Emit && !*p.ok) return;
  const int pg0 = p.ann_poly[g], pg1 = p.ann_poly[g + 1];
  if (pg0 == pg1) {                                 // host run lengths: copied through
    if (Emit) {
      const long long s0 = p.src_off[g], n = p.src_off[g + 1] - s0, o = p.offsets[g];
      for (long long j = (long long)b * kGrThreads + tid; j < n; j += (long long)p.nb * kGrThreads)
        p.counts[o + j] = p.src_counts[s0 + j];
    }
    return;
  }
  const int p0 = b * kGrBand, p1 = min(p0 + kGrBand, h * p.w), nbits = p1 - p0;
  const int nlo = max(0, ceil_div(p0, h) - 1), nhi = (p1 - 1) / h;     // columns whose toggles can land in the band
  const int w0 = tid * kGrPer;
  bool inc = false;                                 // the union's value at pixel p0 - 1
  for (int pg = pg0; pg < pg1; ++pg) {
    const int v0 = p.poly_vert[pg], k = p.poly_vert[pg + 1] - v0;
#pragma unroll
    for (int j = 0; j < kGrPer; ++j) bits[w0 + j] = 0u;
    int par = 0;                                    // toggles below the band seen by this thread, mod 2
    for (int e0 = 0; e0 < k; e0 += kGrThreads) {
      const int e = e0 + tid;
      int cnt = 0;
      if (e < k) {
        const double* a = p.verts + 2 * (size_t)(v0 + e);
        const double* c = p.verts + 2 * (size_t)(v0 + (e + 1 == k ? 0 : e + 1));
        const PolyEdge ed = poly_edge(up5(a[0]), up5(a[1]), up5(c[0]), up5(c[1]), p.w);
        par ^= max(0, min(ed.n1, nlo - 1) - ed.n0 + 1) & 1;
        cnt = max(0, min(ed.n1, nhi) - max(ed.n0, nlo) + 1);
        s_edge[tid] = ed;
      }
      int total;
      s_start[tid] = cta_scan_excl<kGrThreads>(cnt, warp_i, &total);   // its barriers also order the bitmap clear
      __syncthreads();
      for (int it = tid; it < total; it += kGrThreads) {
        int lo = 0, hi = kGrThreads - 1;            // the edge of item it: the last one starting at or before it
        while (lo < hi) {
          const int mid = (lo + hi + 1) >> 1;
          if (s_start[mid] <= it) lo = mid;
          else hi = mid - 1;
        }
        const PolyEdge& ed = s_edge[lo];
        const int a = poly_toggle_index(ed, max(ed.n0, nlo) + it - s_start[lo], h);
        if (a < p0) par ^= 1;
        else if (a < p1) atomicXor(&bits[(a - p0) >> 5], 1u << ((a - p0) & 31));
      }
      __syncthreads();
    }
    const bool odd = __syncthreads_count(par) & 1;  // the polygon's value at pixel p0 - 1
    // prefix XOR over the band from that value, OR-ed into the union (each thread reads and writes its own words)
    unsigned x[kGrPer];
    int cp = 0;
#pragma unroll
    for (int j = 0; j < kGrPer; ++j) { x[j] = bits[w0 + j]; cp ^= __popc(x[j]) & 1; }
    int tot;
    unsigned carry = (unsigned)((cta_scan_excl<kGrThreads>(cp, warp_i, &tot) & 1) ^ (int)odd);
#pragma unroll
    for (int j = 0; j < kGrPer; ++j) {
      unsigned m = x[j];
      m ^= m << 1; m ^= m << 2; m ^= m << 4; m ^= m << 8; m ^= m << 16;
      if (carry) m = ~m;
      carry ^= __popc(x[j]) & 1;
      acc[w0 + j] = pg == pg0 ? m : (acc[w0 + j] | m);
    }
    inc |= odd;
  }
  __syncthreads();                                  // a word's boundary bit 0 reads the word before it
  int nbd = 0, last = -1;
#pragma unroll
  for (int j = 0; j < kGrPer; ++j) {
    const unsigned t = band_edges(acc, w0 + j, inc, nbits);
    nbd += __popc(t);
    if (t) last = p0 + 32 * (w0 + j) + 31 - __clz(t);
  }
  int tot;
  const int excl = cta_scan_excl<kGrThreads>(nbd, warp_i, &tot);
  const int slot = g * p.nb + b;
  if (!Emit) {
    if (nbd && excl + nbd == tot) p.band_last[slot] = last;
    if (tid == 0) {
      p.band_n[slot] = tot;
      if (tot == 0) p.band_last[slot] = -1;
    }
    return;
  }
  int prev = cta_max_excl<kGrThreads>(last, warp_i);
  if (prev < 0) prev = p.band_prev[slot];
  long long o = p.band_base[slot] + excl;
#pragma unroll
  for (int j = 0; j < kGrPer; ++j) {
    unsigned t = band_edges(acc, w0 + j, inc, nbits);
    while (t) {
      const int pos = p0 + 32 * (w0 + j) + __ffs(t) - 1;
      t &= t - 1;
      p.counts[o++] = (unsigned)(pos - prev);
      prev = pos;
    }
  }
}

__global__ void __launch_bounds__(kGrScanThreads) gt_rle_scan_kernel(const GtRleArgs p) {
  __shared__ long long warp_l[kGrScanThreads / 32];
  const int tid = threadIdx.x;
  long long carry = 0;
  for (int g0 = 0; g0 < p.G; g0 += kGrScanThreads) {
    const int g = g0 + tid;
    const bool poly = g < p.G && p.ann_poly[g] != p.ann_poly[g + 1];
    long long runs = 0;
    if (poly) {
      int n = 0, last = 0;
      for (int b = 0; b < p.nb; ++b) {
        const int i = g * p.nb + b;
        p.band_base[i] = n;
        p.band_prev[i] = last;
        n += p.band_n[i];
        if (p.band_last[i] >= 0) last = p.band_last[i];
      }
      p.ann_last[g] = last;
      runs = (long long)n + 1;
    } else if (g < p.G) {
      runs = p.src_off[g + 1] - p.src_off[g];
    }
    long long tot;
    const long long o = carry + cta_scan_excl<kGrScanThreads>(runs, warp_l, &tot);
    if (g < p.G) p.offsets[g] = o;
    if (poly)
      for (int b = 0; b < p.nb; ++b) p.band_base[g * p.nb + b] += o;
    carry += tot;
  }
  const bool ok = carry <= p.cap;
  if (tid == 0) {
    *p.ok = ok;
    p.offsets[p.G] = ok ? carry : 0;
    if (!ok) atomicOr(p.err, UPSNET_GT_RLE_E_CAPACITY);
  }
  __syncthreads();
  const long long hw = (long long)p.h * p.w;
  for (int g = tid; g < p.G; g += kGrScanThreads) {
    if (!ok) p.offsets[g] = 0;
    else if (p.ann_poly[g] != p.ann_poly[g + 1]) p.counts[p.offsets[g + 1] - 1] = (unsigned)(hw - p.ann_last[g]);
  }
}

inline size_t gt_rle_layout(int G, int nb, void* base, GtRleArgs& p) {
  WsCarve c(base);
  const size_t n = (size_t)G * nb;
  p.band_n = c.take<int>(n);
  p.band_last = c.take<int>(n);
  p.band_prev = c.take<int>(n);
  p.band_base = c.take<long long>(n);
  p.ann_last = c.take<int>(G);
  p.ok = c.take<int>(1);
  return c.bytes();
}

inline int gt_rle_bands(int h, int w) { return (int)(((long long)h * w + kGrBand - 1) / kGrBand); }

}  // namespace ups

extern "C" int upsnet_gt_rle_workspace_bytes(int num_anns, int h, int w, size_t* bytes) {
  if (!bytes || num_anns < 0 || h <= 0 || w <= 0) return UPSNET_E_BADARG;
  if ((long long)h * w >= (1ll << 31) || num_anns > 65535) return UPSNET_E_UNSUPPORTED;
  ups::GtRleArgs p{};
  *bytes = ups::gt_rle_layout(num_anns, ups::gt_rle_bands(h, w), nullptr, p);
  return 0;
}

extern "C" int upsnet_gt_rle(int h, int w, int num_anns, const int* ann_poly, const int* poly_vert, const double* verts,
                             const int64_t* src_offsets, const uint32_t* src_counts, uint32_t* gt_counts,
                             long long capacity, int64_t* gt_offsets, int* err, void* workspace, size_t workspace_bytes,
                             void* stream) {
  using namespace ups;
  if (num_anns < 0 || h <= 0 || w <= 0 || capacity < 0) return UPSNET_E_BADARG;
  if (!ann_poly || !poly_vert || !src_offsets || !gt_offsets || !err || (capacity > 0 && !gt_counts)) return UPSNET_E_BADARG;
  if ((long long)h * w >= (1ll << 31) || num_anns > 65535) return UPSNET_E_UNSUPPORTED;
  GtRleArgs p{};
  p.h = h; p.w = w; p.G = num_anns; p.nb = gt_rle_bands(h, w);
  if (!workspace || workspace_bytes < gt_rle_layout(num_anns, p.nb, workspace, p)) return UPSNET_E_WORKSPACE;
  p.ann_poly = ann_poly; p.poly_vert = poly_vert; p.verts = verts;
  p.src_off = (const long long*)src_offsets; p.src_counts = src_counts;
  p.counts = gt_counts; p.cap = capacity; p.offsets = (long long*)gt_offsets; p.err = err;
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid(p.nb, num_anns);
  if (num_anns > 0) {
    gt_rle_band_kernel<false><<<grid, kGrThreads, 0, st>>>(p);
    UPS_CHECK_LAUNCH();
  }
  gt_rle_scan_kernel<<<1, kGrScanThreads, 0, st>>>(p);
  UPS_CHECK_LAUNCH();
  if (num_anns > 0) {
    gt_rle_band_kernel<true><<<grid, kGrThreads, 0, st>>>(p);
    UPS_CHECK_LAUNCH();
  }
  return 0;
}
