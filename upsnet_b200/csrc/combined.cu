// combined.cu -- the combined panoptic result (heuristic merge of the instance output with the semantic head), device
// resident (SURVEY section 8f, the second panoptic producer next to upsnet_unified_pan_result):
//
//  * combined_decide_kernel, block 0: the serial decision in score order.  It compacts the detections the merge looks
//    at (class in [1, num_classes), score >= score_threshold), ranks them by (score desc, class desc, index desc) and
//    walks them one at a time.  Per detection the whole CTA scans its COCO run lengths, counts the mask's pixels (area)
//    and those not yet claimed (remain) over a column-major occupancy bitmap, applies the keep test in float32 and, on
//    keep, claims the free pixels: their bits are set and the (class, instance) byte pair goes into a column-major owner
//    map.  Long runs of ones are cut into 256-pixel pieces, so a full-height mask spreads over every thread.
//  * combined_decide_kernel, blocks 1..: the 256-bin histogram of the semantic map (for the stuff area limit), run
//    concurrently with block 0 in the same launch.
//  * combined_merge_kernel: one 32x32 tile per CTA.  The owner map is transposed through shared memory, and the uint8
//    [H,W,3] map is written row-major: stuff classes under the area limit -> 255, thing / void pixels without an instance
//    -> 255, instance pixels -> (class + id_last_stuff, instance number).
// Masks are never decoded to [H,W] images.  The keep test is the reference's float32 arithmetic: remain and area are exact
// integers (H*W <= 2^24), and the ratio is one correctly rounded float32 division.
#include <cub/block/block_scan.cuh>

#include "common.cuh"
#include "cta.cuh"

namespace ups {

constexpr int kCbThreads = 512;
constexpr int kCbMaxDet = UPSNET_COMBINED_MAX_DET;
constexpr unsigned kCbPiece = 256;                        // pixels per work item of the decide pass (8 bitmap words)
constexpr int kCbTile = 32;

struct CombinedArgs {
  const unsigned char* sem8; const long long* sem64; int H, W;
  const float* scores; const long long* cls; int n; const int* n_dev;
  const unsigned* counts; int cap; const int* run_len;
  int id_last, num_classes; float score_thr, frac_thr; int stuff_limit;
  int* err; unsigned* bits; unsigned short* owner; int* hist;
};

using CbScan = cub::BlockScan<unsigned long long, kCbThreads>;

struct CbSmem {
  unsigned long long key[kCbMaxDet];                      // (score, class, index): descending = the merge order
  short order[kCbMaxDet];                                 // detection of rank r
  unsigned long long start[kCbThreads];                   // first pixel of the chunk's run j (clamped to H*W)
  unsigned len[kCbThreads], poff[kCbThreads];             // pixels of run j if it is a run of ones, else 0; first piece
  unsigned inst[256];                                     // idx_ins_array: kept instances per class
  typename CbScan::TempStorage scan;
  unsigned long long red[2][kCbThreads / 32];
  int nv, keep, err;
  unsigned pieces;
  int hist[256];
};

__device__ __forceinline__ unsigned cb_sem(const CombinedArgs& p, size_t i) {
  return p.sem8 ? (unsigned)p.sem8[i] : (unsigned)(unsigned char)p.sem64[i];
}

// Loads and scans the chunk of run lengths [base, base + kCbThreads) of one detection into shared memory; `carry` is the
// pixel position at the chunk's start (every thread holds it and advances it).
__device__ __forceinline__ void cb_load_chunk(CbSmem& s, const unsigned* __restrict__ cnt, int len, int base,
                                              unsigned long long& carry, unsigned long long HW) {
  const int tid = threadIdx.x, j = base + tid;
  const unsigned long long c = j < len ? (unsigned long long)cnt[j] : 0ull;
  const bool ones = (j & 1) && j < len;
  unsigned long long excl, tot, pexcl, ptot;
  CbScan(s.scan).ExclusiveSum(c, excl, tot);
  const unsigned long long st = min(carry + excl, HW), en = min(carry + excl + c, HW);   // in bounds even for bad input
  const unsigned ln = ones ? (unsigned)(en - st) : 0u;
  __syncthreads();
  CbScan(s.scan).ExclusiveSum((unsigned long long)((ln + kCbPiece - 1) / kCbPiece), pexcl, ptot);
  s.start[tid] = st;
  s.len[tid] = ln;
  s.poff[tid] = (unsigned)pexcl;
  if (tid == 0) s.pieces = (unsigned)ptot;
  carry += tot;
  __syncthreads();
}

// Piece q of the loaded chunk: the run holding it (last run whose first piece is <= q) and its pixel range [ps, pe).
__device__ __forceinline__ void cb_piece(const CbSmem& s, unsigned q, unsigned& ps, unsigned& pe) {
  int lo = 0, hi = kCbThreads;                            // first run with poff > q, minus one
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (s.poff[mid] <= q) lo = mid + 1; else hi = mid; }
  const int r = lo - 1;
  ps = (unsigned)s.start[r] + (q - s.poff[r]) * kCbPiece;
  pe = min(ps + kCbPiece, (unsigned)s.start[r] + s.len[r]);
}

__device__ __forceinline__ unsigned cb_word_mask(unsigned ps, unsigned pe, unsigned w) {
  const unsigned lo = max(ps, w << 5) - (w << 5), hi = min(pe, (w << 5) + 32u) - (w << 5);
  return (hi >= 32u ? ~0u : (1u << hi) - 1u) & ~((1u << lo) - 1u);
}

__device__ void combined_decide(const CombinedArgs& p, CbSmem& s) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned long long HW = (unsigned long long)p.H * p.W;
  const int n = p.n_dev ? min(*p.n_dev, p.n) : p.n;
  if (tid == 0) { s.nv = 0; s.err = 0; }
  for (int c = tid; c < 256; c += kCbThreads) s.inst[c] = 0u;
  __syncthreads();
  if (n > kCbMaxDet) {
    if (tid == 0) atomicOr(p.err, UPSNET_COMBINED_E_DET_COUNT);
    return;
  }
  // the detections the merge looks at; their slot order does not matter, the ranking below orders them
  for (int d = tid; d < n; d += kCbThreads) {
    const long long c = p.cls[d];
    const float sc = p.scores[d];
    if (c < 1 || c >= p.num_classes || sc < p.score_thr) continue;
    // -0 -> +0; one NaN (numpy sorts every NaN last)
    const unsigned u = orderable(sc != sc ? __uint_as_float(0x7fc00000u) : sc + 0.0f);
    s.key[atomicAdd(&s.nv, 1)] = ((unsigned long long)u << 32) | ((unsigned long long)c << 11) | (unsigned long long)d;
  }
  __syncthreads();
  const int nv = s.nv;
  // np.argsort(score, kind='stable')[::-1] over the class-ascending concatenation: keys are distinct, rank = number above
  for (int i = tid; i < nv; i += kCbThreads) {
    const unsigned long long k = s.key[i];
    int r = 0;
    for (int j = 0; j < nv; ++j) r += s.key[j] > k;
    s.order[r] = (short)(k & 2047u);
  }
  __syncthreads();
  for (int r = 0; r < nv; ++r) {
    const int d = s.order[r], len = p.run_len[d];
    if (len < 0 || len > p.cap) {                         // im_post_rle overflowed its buffer: runs unknown
      if (tid == 0) s.err |= UPSNET_COMBINED_E_RUN_LEN;
      continue;
    }
    const unsigned* cnt = p.counts + (size_t)d * p.cap;
    const bool single = len <= kCbThreads;
    unsigned long long carry = 0, remain = 0, area = 0;
    for (int base = 0; base < max(len, 1); base += kCbThreads) {
      cb_load_chunk(s, cnt, len, base, carry, HW);
      for (unsigned q = tid; q < s.pieces; q += kCbThreads) {
        unsigned ps, pe;
        cb_piece(s, q, ps, pe);
        area += pe - ps;
        for (unsigned w = ps >> 5; w <= (pe - 1) >> 5; ++w) remain += __popc(cb_word_mask(ps, pe, w) & ~__ldcg(p.bits + w));
      }
      __syncthreads();
    }
    for (int o = 16; o; o >>= 1) {
      remain += __shfl_xor_sync(0xffffffffu, remain, o);
      area += __shfl_xor_sync(0xffffffffu, area, o);
    }
    if (lane == 0) { s.red[0][warp] = remain; s.red[1][warp] = area; }
    __syncthreads();
    if (tid == 0) {
      unsigned long long rem = 0, ar = 0;
      for (int w = 0; w < kCbThreads / 32; ++w) { rem += s.red[0][w]; ar += s.red[1][w]; }
      int keep = 0;
      if (carry != HW) {
        s.err |= UPSNET_COMBINED_E_RLE_SIZE;
      } else if (ar && __fdiv_rn((float)rem, (float)ar) >= p.frac_thr) {
        const int c = (int)p.cls[d];
        const unsigned inst = ++s.inst[c - 1] & 255u;     // uint32 counter stored into the uint8 instance map
        if (inst) keep = (int)((((unsigned)(c + p.id_last) & 255u) << 8) | inst);
      }
      s.keep = keep;
    }
    __syncthreads();
    const unsigned short v = (unsigned short)s.keep;
    if (!v) continue;                                     // skipped, or the 256th instance of a class (pixels stay free)
    carry = 0;
    for (int base = 0; base < len; base += kCbThreads) {
      if (!single) cb_load_chunk(s, cnt, len, base, carry, HW);
      for (unsigned q = tid; q < s.pieces; q += kCbThreads) {
        unsigned ps, pe;
        cb_piece(s, q, ps, pe);
        for (unsigned w = ps >> 5; w <= (pe - 1) >> 5; ++w) {
          unsigned nb = cb_word_mask(ps, pe, w) & ~__ldcg(p.bits + w);
          if (!nb) continue;
          atomicOr(p.bits + w, nb);                       // other threads only touch other bits of this word
          if (nb == ~0u) {                                // the word's 32 owners are 64 aligned bytes: four 16-byte stores
            const unsigned vv = v | ((unsigned)v << 16);
            uint4* o4 = reinterpret_cast<uint4*>(p.owner + (w << 5));
#pragma unroll
            for (int k = 0; k < 4; ++k) o4[k] = make_uint4(vv, vv, vv, vv);
          } else {
            for (; nb; nb &= nb - 1u) p.owner[(w << 5) + (unsigned)(__ffs(nb) - 1)] = v;
          }
        }
      }
      __syncthreads();
    }
  }
  if (tid == 0 && s.err) atomicOr(p.err, s.err);
}

__global__ void __launch_bounds__(kCbThreads)
combined_decide_kernel(const __grid_constant__ CombinedArgs p) {
  __shared__ CbSmem s;
  if (blockIdx.x == 0) { combined_decide(p, s); return; }
  // semantic class histogram (uint8-wrapped values), shared-memory bins flushed once per block
  for (int c = threadIdx.x; c < 256; c += kCbThreads) s.hist[c] = 0;
  __syncthreads();
  const size_t HW = (size_t)p.H * p.W, stride = (size_t)(gridDim.x - 1) * kCbThreads;
  for (size_t i = (size_t)(blockIdx.x - 1) * kCbThreads + threadIdx.x; i < HW; i += stride) atomicAdd(&s.hist[cb_sem(p, i)], 1);
  __syncthreads();
  for (int c = threadIdx.x; c < 256; c += kCbThreads)
    if (s.hist[c]) atomicAdd(p.hist + c, s.hist[c]);
}

__global__ void __launch_bounds__(kCbTile * 8)
combined_merge_kernel(const __grid_constant__ CombinedArgs p, unsigned char* __restrict__ out) {
  __shared__ unsigned short tile[kCbTile][kCbTile + 1];  // [column][row]
  __shared__ unsigned char stuff_void[256];
  const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kCbTile + tx;
  const int x0 = blockIdx.x * kCbTile, y0 = blockIdx.y * kCbTile;
  for (int c = tid; c < 256; c += kCbTile * 8) stuff_void[c] = c <= p.id_last && p.hist[c] < p.stuff_limit;
  for (int i = ty; i < kCbTile; i += 8) {                 // column-major owner map: 32 consecutive rows of column x
    const int x = x0 + i, y = y0 + tx;
    unsigned short v = 0;
    if (x < p.W && y < p.H) {
      const unsigned q = (unsigned)x * p.H + y;
      if ((p.bits[q >> 5] >> (q & 31)) & 1u) v = p.owner[q];
    }
    tile[i][tx] = v;
  }
  __syncthreads();
  for (int i = ty; i < kCbTile; i += 8) {
    const int y = y0 + i, x = x0 + tx;
    if (x >= p.W || y >= p.H) continue;
    const size_t o = (size_t)y * p.W + x;
    const unsigned sem = cb_sem(p, o), own = tile[tx][i];
    unsigned c0 = stuff_void[sem] ? 255u : sem;           // stuff area limit
    if (own) c0 = own >> 8;                               // instance pixel: its class + id_last_stuff
    else if ((int)c0 > p.id_last) c0 = 255u;              // thing (or void) class without an instance
    out[3 * o] = (unsigned char)c0;
    out[3 * o + 1] = (unsigned char)(own & 255u);
    out[3 * o + 2] = 0;
  }
}

inline size_t cb_layout(int H, int W, void* base, CombinedArgs& p) {
  const size_t HW = (size_t)H * W;
  WsCarve c(base);
  p.hist = c.take<int>(256);
  p.bits = c.take<unsigned>((HW + 31) / 32);
  p.owner = c.take<unsigned short>(HW);
  return c.bytes();
}

}  // namespace ups

extern "C" int upsnet_combined_pan_workspace_bytes(int n, int H, int W, size_t* bytes) {
  if (!bytes || n < 0 || H < 1 || W < 1 || (long long)H * W > (1ll << 24)) return UPSNET_E_BADARG;
  ups::CombinedArgs p{};
  *bytes = ups::cb_layout(H, W, nullptr, p);
  return 0;
}

extern "C" int upsnet_combined_pan_result(const void* sem, int sem_elem_size, int H, int W, const float* scores,
                                          const int64_t* cls_inds, int n, const int* n_dev, const uint32_t* counts, int cap,
                                          const int* run_len, int num_seg_classes, int num_classes, float score_threshold,
                                          float fraction_threshold, int stuff_area_limit, unsigned char* pan_2ch, int* err,
                                          void* workspace, size_t workspace_bytes, void* stream) {
  using namespace ups;
  if (!sem || (sem_elem_size != 1 && sem_elem_size != 8) || !pan_2ch || !err) return UPSNET_E_BADARG;
  if (H < 1 || W < 1 || (long long)H * W > (1ll << 24) || n < 0) return UPSNET_E_BADARG;
  if (num_classes < 1 || num_classes > 256 || num_seg_classes < num_classes || num_seg_classes - num_classes > 255)
    return UPSNET_E_BADARG;
  if (n > 0 && (!scores || !cls_inds || !counts || !run_len || cap < 1)) return UPSNET_E_BADARG;
  CombinedArgs p{sem_elem_size == 1 ? (const unsigned char*)sem : nullptr,
                 sem_elem_size == 8 ? (const long long*)sem : nullptr, H, W,
                 scores, (const long long*)cls_inds, n, n_dev, counts, cap, run_len,
                 num_seg_classes - num_classes, num_classes, score_threshold, fraction_threshold, stuff_area_limit,
                 err};
  if (!workspace || workspace_bytes < cb_layout(H, W, workspace, p)) return UPSNET_E_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  // histogram + occupancy bitmap (the owner map is read under it)
  UPS_CUDA(cudaMemsetAsync(p.hist, 0, (char*)p.owner - (char*)p.hist, st));
  const int hist_blocks = max(1, min(2 * num_sms(), ceil_div(H * W, kCbThreads * 16)));
  combined_decide_kernel<<<1 + hist_blocks, kCbThreads, 0, st>>>(p);
  UPS_CHECK_LAUNCH();
  combined_merge_kernel<<<dim3(ceil_div(W, kCbTile), ceil_div(H, kCbTile)), dim3(kCbTile, 8), 0, st>>>(p, pan_2ch);
  UPS_CHECK_LAUNCH();
  return 0;
}
