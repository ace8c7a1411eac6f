// panoptic.cu -- fused parameter-free panoptic head for sm_90a.
//
// Restates models/resnet_upsnet.py:223-240 of the reference:
//   MaskRemoval  (operators/modules/mask_removal.py:29-93)  score-ordered overlap pruning
//   SegTerm      (operators/modules/unary_logits.py:78-105) boxed copy of the thing logit
//   void = max(thing logits) - max_i(seg_inst);  cat;  argmax;  void -> 255
// without ever materialising the three [1,k,H,W] fp32 planes (0.8-8 GB each in the reference).
//
// Kernels
//   pan_prep     1 CTA : rank instances by score (counting rank, stable), integer geometry.
//   pan_bits     whole GPU: the resized-logit > 0 bit mask of EVERY instance (no dependence on the keep
//                decisions), packed 32 pixels / word over the instance's paste window, + |mask| by popc.
//   pan_decide   1 CTA per thing class: serial over that class's instances in score order -- the only
//                inherently sequential part (mask_removal.py:66-86) -- now just popc(bits & occupied) over
//                the window words, the float64 ratio test, and occupied |= bits for the kept ones.
//   pan_compact  1 CTA : kept list in score order (ballot prefix sums), k==0 fallback.
//   pan_fuse     CTA per 128x8 pixel tile: bins the kept instances against the tile, then every
//                thread streams the S semantic logits of 4 consecutive pixels (float4, coalesced)
//                and runs the ordered argmax over [stuff | instances | void].
// pan_fuse is the bandwidth kernel: algorithmic bytes = 4*S*H*W + 8*H*W (+8*H*W with
// sem_labels) + n*(3136+24); see DESIGN.md.  Arithmetic of the 28x28 -> (w,h) resize is the
// oracle-of-record formula (oracle/upsnet_oracle.c resized_logit) in un-fused fp32 (_rn
// intrinsics) so label maps are bit-exact.
#include "common.cuh"
#include "cta.cuh"
#include "up4.cuh"

namespace ups {

constexpr int kMaskS = 28;
constexpr int kMaskElems = kMaskS * kMaskS;
constexpr int kMaxList = 2048;   // max instances per call (per-tile / per-class uint16 lists)
constexpr int kMaxRounds = 64;
constexpr long long kBitsBudget = 16ll << 20;   // words (64 MB) of instance bit windows resident at a time

// per-instance integer geometry, SoA with stride n (indexed by ORIGINAL instance id)
struct PanGeom {
  int* bx0; int* by0; int* w; int* h;        // truncated box origin and size
  int* gx0; int* gy0; int* gx1; int* gy1;    // mask paste window (image coords, clamped)
  int* sx0; int* sy0; int* sx1; int* sy1;    // SegTerm window (python-slice clamped)
  int* cls;                                  // 1-based thing class (0 = dummy)
};

struct PanWorkspace {
  int* order;       // [n]  rank -> original index (score desc, stable)
  int* kept_flag;   // [n]  by rank
  int* kept_list;   // [n]  compacted: original indices in score order
  int* meta;        // [4]  k, zero_mask, ...
  PanGeom g;
  unsigned int* occ;      // [num_thing][H][Ww]  occupancy bit planes
  long long* off;         // [n]  by rank: word offset of the instance's bit window (exclusive scan of window sizes)
  int* msum;              // [n]  by rank: |mask| (popc over the window)
  int* round_lo;          // [kMaxRounds + 1]  first rank of every bit-buffer round (ranks of a round are contiguous)
  unsigned int* bits;     // [budget + H*Ww]  bit windows of the instances of the current round
  long long budget;       // words per round
  int rounds;
};

// avail = 0: the preferred layout (all bit windows resident, up to kBitsBudget).  avail > 0: the caller's workspace size
// -- the bit-window budget shrinks to what fits (more rounds of consecutive ranks), so the round structure is a RUNTIME
// property of the call; returns 0 when not even the minimum (one window, or all / kMaxRounds words) fits.
static inline size_t pan_ws_layout(int n, int H, int W, int num_thing, PanWorkspace& ws,
                                                void* base, size_t avail = 0) {
  const int nn = n > 0 ? n : 1;
  WsCarve c(base);
  ws.order = c.take<int>(nn);
  ws.kept_flag = c.take<int>(nn);
  ws.kept_list = c.take<int>(nn);
  ws.meta = c.take<int>(4);
  int* g = c.take<int>((size_t)nn * 13);
  if (g) {
    ws.g.bx0 = g; ws.g.by0 = g + nn; ws.g.w = g + 2 * nn; ws.g.h = g + 3 * nn;
    ws.g.gx0 = g + 4 * nn; ws.g.gy0 = g + 5 * nn; ws.g.gx1 = g + 6 * nn; ws.g.gy1 = g + 7 * nn;
    ws.g.sx0 = g + 8 * nn; ws.g.sy0 = g + 9 * nn; ws.g.sx1 = g + 10 * nn; ws.g.sy1 = g + 11 * nn;
    ws.g.cls = g + 12 * nn;
  }
  const int Ww = ceil_div(W, 32);
  ws.occ = c.take<unsigned int>((size_t)num_thing * H * Ww);
  ws.off = c.take<long long>(nn);
  ws.msum = c.take<int>(nn);
  ws.round_lo = c.take<int>(kMaxRounds + 1);
  // bit windows: every instance needs at most one full plane (H*Ww words).  All of them are resident when they
  // fit the budget, otherwise the instances are processed in rounds of consecutive ranks.
  const long long win = (long long)H * Ww, all = win * nn;
  long long budget = all < kBitsBudget ? all : kBitsBudget;
  if (avail) {
    const long long fit = ((long long)avail - (long long)c.bytes()) / (long long)sizeof(unsigned int) - win - 64;
    if (fit < budget) budget = fit;
    if (budget < win || (all + budget - 1) / budget > kMaxRounds) return 0;
  }
  if ((all + budget - 1) / budget > kMaxRounds) budget = (all + kMaxRounds - 1) / kMaxRounds;
  if (budget < win) budget = win;
  ws.rounds = (int)((all + budget - 1) / budget);
  ws.budget = budget;
  ws.bits = c.take<unsigned int>((size_t)(budget + win));
  return c.bytes();
}

// ---- resize coefficients: oracle resize_coef_x / resize_coef_y, un-fused ----
__device__ __forceinline__ void coef_x(int d, int n_dst, int& s, float& f) {
  const double scale = __ddiv_rn((double)kMaskS, (double)n_dst);
  float fv = (float)__dadd_rn(__dmul_rn((double)d + 0.5, scale), -0.5);
  int sv = (int)floorf(fv);
  fv = __fsub_rn(fv, (float)sv);
  if (sv < 0) { sv = 0; fv = 0.f; }
  if (sv >= kMaskS - 1) { sv = kMaskS - 1; fv = 0.f; }
  s = sv; f = fv;
}
__device__ __forceinline__ void coef_y(int d, int n_dst, int& s, float& f) {
  const double scale = __ddiv_rn((double)kMaskS, (double)n_dst);
  float fv = (float)__dadd_rn(__dmul_rn((double)d + 0.5, scale), -0.5);
  const int sv = (int)floorf(fv);
  s = sv; f = __fsub_rn(fv, (float)sv);
}
__device__ __forceinline__ float blend(const float* __restrict__ S, int sx, float fx, int sy, float fy) {
  const int sx1 = min(sx + 1, kMaskS - 1);
  const int y0 = min(max(sy, 0), kMaskS - 1), y1 = min(max(sy + 1, 0), kMaskS - 1);
  const float a0 = __fsub_rn(1.f, fx), a1 = fx, b0 = __fsub_rn(1.f, fy), b1 = fy;
  const float h0 = __fadd_rn(__fmul_rn(S[y0 * kMaskS + sx], a0), __fmul_rn(S[y0 * kMaskS + sx1], a1));
  const float h1 = __fadd_rn(__fmul_rn(S[y1 * kMaskS + sx], a0), __fmul_rn(S[y1 * kMaskS + sx1], a1));
  return __fadd_rn(__fmul_rn(h0, b0), __fmul_rn(h1, b1));
}

// ------------------------------------------------------------------------------------------
constexpr int kPrepThreads = 1024;

__global__ void __launch_bounds__(kPrepThreads)
pan_prep_kernel(const float* __restrict__ boxes, const float* __restrict__ prob,
                const int64_t* __restrict__ cls_idx, int n_max, const int* __restrict__ n_dev, int H, int W,
                PanWorkspace ws) {
  const int n = n_dev ? max(min(*n_dev, n_max), 1) : n_max;   // device-side instance count (static-shape engine)
  if (threadIdx.x == 0) ws.meta[2] = n;
  __shared__ float s_prob[kMaxList];            // n <= kMaxList (checked by the entry point): the rank loop reads shared memory
  for (int i = threadIdx.x; i < n; i += kPrepThreads) s_prob[i] = prob[i];
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += kPrepThreads) {
    const float p = s_prob[i];
    int rank = 0;
    for (int j = 0; j < n; ++j) {
      const float q = s_prob[j];
      rank += (q > p) || (q == p && j < i);
    }
    ws.order[rank] = i;
    const float* b = boxes + (size_t)i * 4;
    const int bx0 = (int)b[0], by0 = (int)b[1], bx1 = (int)b[2], by1 = (int)b[3];  // astype(int32)
    const int w = max(bx1 - bx0 + 1, 1), h = max(by1 - by0 + 1, 1);
    ws.g.bx0[i] = bx0; ws.g.by0[i] = by0; ws.g.w[i] = w; ws.g.h[i] = h;
    ws.g.gx0[i] = max(bx0, 0); ws.g.gx1[i] = min(bx1 + 1, W);
    ws.g.gy0[i] = max(by0, 0); ws.g.gy1[i] = min(by1 + 1, H);
    const int c = (int)cls_idx[i];
    // unary_logits.py:92-103: boxes*4.0*0.25 is exact in binary fp; int() truncates, round() is
    // numpy half-to-even (rintf); python slices clamp to the array extent.
    const float fb0 = __fmul_rn(__fmul_rn(b[0], 4.0f), 0.25f), fb1 = __fmul_rn(__fmul_rn(b[1], 4.0f), 0.25f);
    const float fb2 = __fmul_rn(__fmul_rn(b[2], 4.0f), 0.25f), fb3 = __fmul_rn(__fmul_rn(b[3], 4.0f), 0.25f);
    int sx0 = min((int)fb0, W), sy0 = min((int)fb1, H);
    int sx1 = min((int)(rintf(fb2) + 1.f), W), sy1 = min((int)(rintf(fb3) + 1.f), H);
    if (c == 0) { sx1 = sx0; sy1 = sy0; }
    ws.g.sx0[i] = sx0; ws.g.sy0[i] = sy0; ws.g.sx1[i] = sx1; ws.g.sy1[i] = sy1;
    ws.g.cls[i] = c;
  }
  // ---- bit-window sizes by rank -> exclusive scan -> word offsets and round boundaries ----
  __shared__ long long warp_sums[kPrepThreads / 32];
  long long carry = 0;
  for (int q = threadIdx.x; q <= kMaxRounds; q += kPrepThreads) ws.round_lo[q] = n;
  __syncthreads();   // order[] and the geometry are complete
  for (int base = 0; base < n; base += kPrepThreads) {
    const int r = base + threadIdx.x;
    long long sz = 0;
    if (r < n) {
      const int i = ws.order[r];
      const int x0 = ws.g.gx0[i], x1 = ws.g.gx1[i], y0 = ws.g.gy0[i], y1 = ws.g.gy1[i];
      sz = (long long)max(((x1 + 31) >> 5) - (x0 >> 5), 0) * max(y1 - y0, 0);
    }
    long long tot;
    const long long excl = cta_scan_excl<kPrepThreads>(sz, warp_sums, &tot);
    if (r < n) {
      ws.off[r] = carry + excl;
      ws.msum[r] = 0;
    }
    carry += tot;
  }
  __syncthreads();   // off[] is complete
  // round boundaries: rank r opens round q when it is the first rank whose start offset falls in [q*budget, ...)
  for (int r = threadIdx.x; r < n; r += kPrepThreads) {
    const int rq = (int)(ws.off[r] / ws.budget);
    if (r == 0 || (int)(ws.off[r - 1] / ws.budget) != rq) ws.round_lo[rq] = r;
  }
}

__device__ __forceinline__ void cp_async4(float* dst_smem, const float* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all_() {
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
}

// The mask bits of every instance of round `rq`: grid (kBitsChunks, n_max), CTA = (chunk of the window rows x words,
// rank).  The column coefficients of the 28 -> w resize (float64 scale, oracle resize_coef_x) are computed once per
// CTA into shared memory instead of once per pixel.
constexpr int kBitsChunks = 8, kBitsThreads = 256, kColCap = 2048;
__global__ void __launch_bounds__(kBitsThreads)
pan_bits_kernel(const float* __restrict__ mask_logit, int n_max, const int* __restrict__ n_dev, int rq, PanWorkspace ws) {
  const int n = n_dev ? max(min(*n_dev, n_max), 1) : n_max;
  const int r = blockIdx.y;
  if (r >= n || r < ws.round_lo[rq] || r >= ws.round_lo[rq + 1]) return;
  if (n == 1 && ws.g.cls[0] == 0) return;   // MaskROI's dummy detection
  __shared__ float S[kMaskElems];
  __shared__ float s_fx[kColCap];
  __shared__ unsigned char s_sx[kColCap];
  const int i = ws.order[r];
  const int bx0 = ws.g.bx0[i], by0 = ws.g.by0[i], w = ws.g.w[i], h = ws.g.h[i];
  const int x0 = ws.g.gx0[i], x1 = ws.g.gx1[i], y0 = ws.g.gy0[i], y1 = ws.g.gy1[i];
  const int wx0 = x0 >> 5, wx1 = (x1 + 31) >> 5;
  const int nwc = max(wx1 - wx0, 0), rows = max(y1 - y0, 0);
  const int items = nwc * rows;
  const int per = (items + kBitsChunks - 1) / kBitsChunks;
  const int it0 = blockIdx.x * per, it1 = min(it0 + per, items);
  if (it0 >= it1) return;
  for (int t = threadIdx.x; t < kMaskElems; t += kBitsThreads) S[t] = __ldg(mask_logit + (size_t)i * kMaskElems + t);
  const int ncol = x1 - x0;
  const bool tab = ncol <= kColCap;
  if (tab)
    for (int t = threadIdx.x; t < ncol; t += kBitsThreads) {
      const int dx = x0 + t - bx0;
      int sx = 0; float fx = 0.f;
      if (dx >= 0 && dx < w) coef_x(dx, w, sx, fx);
      s_sx[t] = (unsigned char)sx; s_fx[t] = fx;
    }
  __syncthreads();
  unsigned int* bits = ws.bits + (ws.off[r] - (long long)rq * ws.budget);
  unsigned int my_sum = 0;
  for (int item = it0 + threadIdx.x; item < it1; item += kBitsThreads) {
    const int wy = y0 + item / nwc, wc = wx0 + item % nwc;
    unsigned int word = 0;
    const int dy = wy - by0;
    if (dy >= 0 && dy < h) {
      int sy; float fy;
      coef_y(dy, h, sy, fy);
      const int xa = max(wc * 32, x0), xb = min(wc * 32 + 32, x1);
      for (int x = xa; x < xb; ++x) {
        const int dx = x - bx0;
        if (dx >= 0 && dx < w) {
          int sx; float fx;
          if (tab) { sx = s_sx[x - x0]; fx = s_fx[x - x0]; } else coef_x(dx, w, sx, fx);
          if (blend(S, sx, fx, sy, fy) > 0.f) word |= 1u << (x & 31);
        }
      }
    }
    bits[item] = word;
    my_sum += __popc(word);
  }
#pragma unroll
  for (int sh = 16; sh > 0; sh >>= 1) my_sum += __shfl_xor_sync(0xffffffffu, my_sum, sh);
  if ((threadIdx.x & 31) == 0 && my_sum) atomicAdd(&ws.msum[r], (int)my_sum);
}

// One CTA per thing class (blockIdx.x = class-1): the keep decision of an instance depends only on the earlier
// kept instances of the SAME class, so classes run concurrently and each CTA walks its class's instances of the
// round in score order: |mask & occupied| by popc over the precomputed window words, the float64 ratio test
// (mask_removal.py:82), occupied |= mask for the kept ones.
constexpr int kDecideThreads = 1024;

__global__ void __launch_bounds__(kDecideThreads)
pan_decide_kernel(int n_max, const int* __restrict__ n_dev, int H, int W, double fraction_threshold, int rq,
                  PanWorkspace ws) {
  const int n = n_dev ? max(min(*n_dev, n_max), 1) : n_max;
  __shared__ unsigned short list[kMaxList];   // ranks (score order) of this class's instances in this round
  __shared__ int s_warp_cnt[32];
  const int c = blockIdx.x;  // 0-based class
  const int Ww = ceil_div(W, 32);
  unsigned int* occ = ws.occ + (size_t)c * H * Ww;
  const int lane = threadIdx.x & 31;
  if (n == 1 && ws.g.cls[0] == 0) return;  // MaskROI's dummy detection: mask_removal.py:55-57
  const int r_lo = ws.round_lo[rq], r_hi = min(ws.round_lo[rq + 1], n);
  if (r_lo >= r_hi) return;

  // ---- ordered list of the ranks that belong to this class ----
  int cnt = 0;
  for (int base = r_lo; base < r_hi; base += kDecideThreads) {
    const int r = base + threadIdx.x;
    const bool mine = r < r_hi && ws.g.cls[ws.order[r]] - 1 == c;
    int tot;
    const int rank = cta_ballot_rank<kDecideThreads>(mine, s_warp_cnt, &tot);
    if (mine) list[cnt + rank] = (unsigned short)r;
    cnt += tot;
  }
  __syncthreads();   // list is complete
  // per-instance metadata of the whole class list staged in (dynamic) shared memory: inside the decision loops nothing but
  // the window words and the occupancy words comes from L2
  extern __shared__ __align__(16) unsigned char s_dyn[];
  int4* s_win = reinterpret_cast<int4*>(s_dyn);                       // (wx0, nwc, y0, rows)    [n_max]
  long long* s_off = reinterpret_cast<long long*>(s_win + n_max);      // word offset in ws.bits  [n_max]
  int* s_msum = reinterpret_cast<int*>(s_off + n_max);                 // |mask|                  [n_max]
  volatile int* s_state = reinterpret_cast<volatile int*>(s_msum + n_max);   // 0 undecided, 1 dropped, 2 kept   [n_max]
  for (int li = threadIdx.x; li < cnt; li += kDecideThreads) {
    const int r = list[li];
    const int i = ws.order[r];
    const int x0 = ws.g.gx0[i], x1 = ws.g.gx1[i], y0 = ws.g.gy0[i], y1 = ws.g.gy1[i];
    const int wx0 = x0 >> 5, nwc = max(((x1 + 31) >> 5) - wx0, 0);
    s_win[li] = make_int4(wx0, nwc, y0, max(y1 - y0, 0));
    s_off[li] = ws.off[r] - (long long)rq * ws.budget;
    s_msum[li] = ws.msum[r];
    s_state[li] = 0;
  }
  __syncthreads();
  // The keep decision of an instance depends on the EARLIER instances of its class only through the occupancy words of its
  // own window (mask_removal.py:62-90): two instances whose word windows are disjoint never see each other.  So the score-
  // ordered chain is only as long as the chain of OVERLAPPING windows: eight groups of 128 threads take the instances round-
  // robin, a group first waits for every earlier overlapping instance to be decided (shared-memory state flags), then does
  // what the serial version did -- popc(window & occupied), the float64 ratio test, occupied |= window -- with group-local
  // barriers.  Disjoint windows share no occupancy word, so concurrent groups never write the same word.  Decisions are
  // identical to the serial order; per-instance latency is unchanged, independent instances overlap.
  // (measured and rejected: one warp per instance -- 32 in flight instead of 8 -- is 4x slower, 191 vs 53 us at n = 100: the
  // item loops of an instance are a chain of L2 round trips per thread, so fewer threads per instance lengthen every link)
  constexpr int kGroup = 128, kGroups = 1024 / kGroup;
  __shared__ unsigned int s_part[kGroups][kGroup / 32];
  const int grp = threadIdx.x / kGroup, gt = threadIdx.x % kGroup, gw = gt >> 5;
  for (int li = grp; li < cnt; li += kGroups) {
    const int r = list[li];
    const int4 win = s_win[li];
    const int wx0 = win.x, nwc = win.y, y0 = win.z, rows = win.w;
    const int items = nwc * rows;
    // ---- dependencies: every earlier instance whose word window intersects this one must have been decided ----
    for (int lj = gt; lj < li; lj += kGroup) {
      const int4 o = s_win[lj];
      const bool hit = o.x < wx0 + nwc && wx0 < o.x + o.y && o.z < y0 + rows && y0 < o.z + o.w && o.y > 0 && o.w > 0 && items > 0;
      if (hit) {
        while (s_state[lj] == 0) { }
      }
    }
    __threadfence_block();                        // acquire side of the state flags: the deciders' occupancy writes are visible
    asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "n"(kGroup) : "memory");
    const unsigned int* __restrict__ bits = ws.bits + s_off[li];
    unsigned int my_ovl = 0;
    for (int item = gt; item < items; item += kGroup) {
      const size_t o = (size_t)(y0 + item / nwc) * Ww + (wx0 + item % nwc);
      my_ovl += __popc(__ldg(bits + item) & __ldcg(occ + o));      // occupancy: L2 (another group's SM-local L1 line may be stale)
    }
#pragma unroll
    for (int sh = 16; sh > 0; sh >>= 1) my_ovl += __shfl_xor_sync(0xffffffffu, my_ovl, sh);
    if (lane == 0) s_part[grp][gw] = my_ovl;
    asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "n"(kGroup) : "memory");
    const unsigned int ov = s_part[grp][0] + s_part[grp][1] + s_part[grp][2] + s_part[grp][3];
    const unsigned int ms = (unsigned int)s_msum[li];
    // mask_removal.py:82: int/int true division (float64) compared with the python float 0.3; decided without the division
    // whenever ov is clear of thr*ms by more than rounding could account for (1e-12 relative >> 2^-52) -- every thread of the
    // group evaluates the same expression on the same operands (fp64 is slow on the SM, but this is 3 flops per thread)
    bool drop;
    {
      const double t = (double)ms * fraction_threshold, dov = (double)ov;
      if (ms == 0) drop = true;
      else if (dov > t * (1.0 + 1e-12)) drop = true;
      else if (dov < t * (1.0 - 1e-12)) drop = false;
      else drop = __ddiv_rn(dov, (double)ms) > fraction_threshold;
    }
    if (!drop) {
      for (int item = gt; item < items; item += kGroup) {
        const unsigned int w = __ldg(bits + item);
        if (w) {
          const size_t o = (size_t)(y0 + item / nwc) * Ww + (wx0 + item % nwc);
          __stcg(occ + o, __ldcg(occ + o) | w);
        }
      }
    }
    __threadfence_block();                        // release: occupancy words before the state flag
    asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "n"(kGroup) : "memory");
    if (gt == 0) {
      ws.kept_flag[r] = drop ? 0 : 1;
      s_state[li] = drop ? 1 : 2;
    }
  }
}

constexpr int kCompactThreads = 1024;

__global__ void __launch_bounds__(kCompactThreads)
pan_compact_kernel(int n_max, const int* __restrict__ n_dev, PanWorkspace ws, int64_t* __restrict__ keep_out,
                   int* __restrict__ k_out) {
  __shared__ int s_wcnt[kCompactThreads / 32];
  const int n = n_dev ? max(min(*n_dev, n_max), 1) : n_max;
  int k = 0;
  for (int base = 0; base < n; base += kCompactThreads) {   // ordered (rank order) compaction
    const int r = base + threadIdx.x;
    const bool kept = r < n && ws.kept_flag[r] != 0;
    int tot;
    const int rank = cta_ballot_rank<kCompactThreads>(kept, s_wcnt, &tot);
    if (kept) {
      const int i = ws.order[r];
      ws.kept_list[k + rank] = i;
      keep_out[k + rank] = i;
    }
    k += tot;
  }
  if (threadIdx.x == 0) {
    int zero_mask = 0;
    if (k == 0) {  // mask_removal.py:89-92 (and :55-57): keep=[0] with an all-zero mask plane
      ws.kept_list[0] = 0; keep_out[0] = 0; k = 1; zero_mask = 1;
    }
    ws.meta[0] = k; ws.meta[1] = zero_mask;
    k_out[0] = k;
  }
}

// ------------------------------------------------------------------------------------------
constexpr int kTileW = 128, kTileH = 8, kFuseThreads = 256;

struct Best { float v; int i; };
__device__ __forceinline__ void feed(Best& b, float v, int i) { if (v > b.v) { b.v = v; b.i = i; } }

// UP4: `fcn` is the quarter-resolution score map [S,H/4,W/4] and the x4 bilinear up-sampling of models/fcn.py:88-101 is
// evaluated on the fly (up4.cuh: the same inlined arithmetic as upsample_bilinear_nchw_kernel, so the logits are bit-identical
// to a materialised fcn_output) -- the 4*S*H*W-byte tensor is neither written nor read: the kernel streams 4*S*H*W/16 bytes.
template <bool UP4>
__global__ void __launch_bounds__(kFuseThreads)
pan_fuse_kernel(const float* __restrict__ fcn, int S, int H, int W, int num_stuff,
                const float* __restrict__ mask_logit, PanWorkspace ws,
                int64_t* __restrict__ labels, int64_t* __restrict__ sem_labels) {
  __shared__ unsigned short list[kMaxList];
  __shared__ int s_first_unlisted;
  __shared__ int s_warp_cnt[kFuseThreads / 32];
  const int k = ws.meta[0], zero_mask = ws.meta[1];
  const int tx0 = blockIdx.x * kTileW, ty0 = blockIdx.y * kTileH;
  const int tx1 = min(tx0 + kTileW, W), ty1 = min(ty0 + kTileH, H);
  if (threadIdx.x == 0) s_first_unlisted = k;
  __syncthreads();
  int n_hit = 0;
  // ---- bin kept instances against this tile (ascending j preserved) ----
  for (int base = 0; base < k; base += kFuseThreads) {
    const int j = base + threadIdx.x;
    bool hit = false;
    if (j < k) {
      const int i = ws.kept_list[j];
      const bool hit_seg = ws.g.sx0[i] < tx1 && ws.g.sx1[i] > tx0 && ws.g.sy0[i] < ty1 && ws.g.sy1[i] > ty0;
      const bool hit_msk = !zero_mask && ws.g.gx0[i] < tx1 && ws.g.gx1[i] > tx0 && ws.g.gy0[i] < ty1 &&
                           ws.g.gy1[i] > ty0;
      hit = hit_seg || hit_msk;
      if (!hit) atomicMin(&s_first_unlisted, j);
    }
    int tot;
    const int pos = n_hit + cta_ballot_rank<kFuseThreads>(hit, s_warp_cnt, &tot);
    if (hit && pos < kMaxList) list[pos] = (unsigned short)j;
    n_hit += tot;
  }
  __syncthreads();   // list and s_first_unlisted are complete
  const int cnt = min(n_hit, kMaxList);
  const int u0 = s_first_unlisted;  // smallest kept index whose windows miss the tile (value 0)
  const bool any_unlisted = u0 < k;

  // ---- per-thread: 4 consecutive pixels of one row ----
  const int x = tx0 + (threadIdx.x & 31) * 4, y = ty0 + (threadIdx.x >> 5);
  if (y >= H || x >= W) return;
  const size_t HW = (size_t)H * W;
  const size_t p = (size_t)y * W + x;
  const bool vec = (x + 3 < W) && ((W & 3) == 0);
  const int npx = vec ? 4 : min(4, W - x);

  const int Hs = H >> 2, Ws = W >> 2, xq = x >> 2;       // UP4: source geometry, source column of this thread's quad
  const size_t HWs = (size_t)Hs * Ws;
  Up4Row urow;
  if (UP4) urow = up4_row(y, Hs);
  Best best[4], sem[4];
  float thing_max[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) { best[q].v = -INFINITY; best[q].i = 0; sem[q].v = -INFINITY; sem[q].i = 0; thing_max[q] = -INFINITY; }
  // channels in batches of 4: the four 16-byte loads of a batch are issued before the first compare
  // (memory-level parallelism: this kernel is the HBM-bound one, 4*S*H*W bytes stream through here once)
  for (int cb = 0; cb < S; cb += 4) {
    float vv[4][4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int c = cb + u;
      if (c < S) {
        if (UP4) {
          const float* pl = fcn + (size_t)c * HWs;
          up4_quad(pl + (size_t)urow.y0 * Ws, pl + (size_t)urow.y1 * Ws, xq, Ws, urow.ly, urow.hy, vv[u]);
        } else if (vec) {
          const float4 t = __ldg((const float4*)(fcn + (size_t)c * HW + p));
          vv[u][0] = t.x; vv[u][1] = t.y; vv[u][2] = t.z; vv[u][3] = t.w;
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q) vv[u][q] = q < npx ? __ldg(fcn + (size_t)c * HW + p + q) : 0.f;
        }
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int c = cb + u;
      if (c >= S) break;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float v = vv[u][q];
        if (c == 0) { best[q].v = v; sem[q].v = v; }
        else {
          if (c < num_stuff) feed(best[q], v, c);
          feed(sem[q], v, c);
        }
        if (c >= num_stuff) thing_max[q] = (c == num_stuff) ? v : fmaxf(thing_max[q], v);
      }
    }
  }
  // ---- instances, ascending kept index; unlisted instances contribute the value 0 at u0 ----
  float inst_max[4];
  bool inst_init[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) { inst_max[q] = 0.f; inst_init[q] = any_unlisted; }
  bool fed_unlisted = !any_unlisted;
  for (int li = 0; li < cnt; ++li) {
    const int j = list[li];
    if (!fed_unlisted && j > u0) {
#pragma unroll
      for (int q = 0; q < 4; ++q) feed(best[q], 0.f, num_stuff + u0);
      fed_unlisted = true;
    }
    const int i = ws.kept_list[j];
    const int sx0 = ws.g.sx0[i], sx1 = ws.g.sx1[i], sy0 = ws.g.sy0[i], sy1 = ws.g.sy1[i];
    const int gx0 = ws.g.gx0[i], gx1 = ws.g.gx1[i], gy0 = ws.g.gy0[i], gy1 = ws.g.gy1[i];
    const int bx0 = ws.g.bx0[i], by0 = ws.g.by0[i], bw = ws.g.w[i], bh = ws.g.h[i];
    const bool row_seg = y >= sy0 && y < sy1;
    const int dy = y - by0;
    const bool row_msk = !zero_mask && y >= gy0 && y < gy1 && dy >= 0 && dy < bh;
    const float* seg_plane = fcn + (size_t)(num_stuff + ws.g.cls[i] - 1) * (UP4 ? HWs : HW) + (UP4 ? (size_t)0 : p);
    float segq[4] = {0.f, 0.f, 0.f, 0.f};
    if (UP4 && row_seg) up4_quad(seg_plane + (size_t)urow.y0 * Ws, seg_plane + (size_t)urow.y1 * Ws, xq, Ws, urow.ly, urow.hy, segq);
    const float* Sm = mask_logit + (size_t)i * kMaskElems;
    int sy = 0; float fy = 0.f;
    if (row_msk) coef_y(dy, bh, sy, fy);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (q >= npx) break;
      const int xx = x + q;
      float seg = 0.f;
      if (row_seg && xx >= sx0 && xx < sx1) seg = UP4 ? segq[q] : __ldg(seg_plane + q);
      float m = 0.f;
      const int dx = xx - bx0;
      if (row_msk && xx >= gx0 && xx < gx1 && dx >= 0 && dx < bw) {
        int sx; float fx;
        coef_x(dx, bw, sx, fx);
        m = blend(Sm, sx, fx, sy, fy);
      }
      feed(best[q], __fadd_rn(seg, m), num_stuff + j);
      if (!inst_init[q]) { inst_max[q] = seg; inst_init[q] = true; } else inst_max[q] = fmaxf(inst_max[q], seg);
    }
  }
  if (!fed_unlisted) {
#pragma unroll
    for (int q = 0; q < 4; ++q) feed(best[q], 0.f, num_stuff + u0);
  }
  long long out[4], semo[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float voidv = __fsub_rn(thing_max[q], inst_max[q]);
    feed(best[q], voidv, num_stuff + k);
    out[q] = (best[q].i == num_stuff + k) ? 255 : best[q].i;
    semo[q] = sem[q].i;
  }
  if (vec) {
    longlong2* o = (longlong2*)(labels + p);
    o[0] = make_longlong2(out[0], out[1]);
    o[1] = make_longlong2(out[2], out[3]);
    if (sem_labels) {
      longlong2* so = (longlong2*)(sem_labels + p);
      so[0] = make_longlong2(semo[0], semo[1]);
      so[1] = make_longlong2(semo[2], semo[3]);
    }
  } else {
    for (int q = 0; q < npx; ++q) { labels[p + q] = out[q]; if (sem_labels) sem_labels[p + q] = semo[q]; }
  }
}

// Materialises MaskRemoval's second output, mask_energy [k,H,W] (mask_removal.py:86): the resized logit
// inside the paste window, 0 elsewhere.  API-parity path only (the fused head never builds these planes).
__global__ void __launch_bounds__(256)
pan_paste_kernel(const float* __restrict__ mask_logit, int H, int W, PanWorkspace ws, float* __restrict__ energy) {
  const int k = ws.meta[0], zero_mask = ws.meta[1];
  const int j = blockIdx.y;
  if (j >= k) return;
  const int i = ws.kept_list[j];
  const int bx0 = ws.g.bx0[i], by0 = ws.g.by0[i], bw = ws.g.w[i], bh = ws.g.h[i];
  const int gx0 = ws.g.gx0[i], gx1 = ws.g.gx1[i], gy0 = ws.g.gy0[i], gy1 = ws.g.gy1[i];
  const float* Sm = mask_logit + (size_t)i * kMaskElems;
  const size_t HW = (size_t)H * W;
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (size_t)gridDim.x * blockDim.x) {
    const int y = (int)(p / W), x = (int)(p - (size_t)y * W);
    float v = 0.f;
    const int dx = x - bx0, dy = y - by0;
    if (!zero_mask && x >= gx0 && x < gx1 && y >= gy0 && y < gy1 && dx >= 0 && dx < bw && dy >= 0 && dy < bh) {
      int sx, sy; float fx, fy;
      coef_x(dx, bw, sx, fx);
      coef_y(dy, bh, sy, fy);
      v = blend(Sm, sx, fx, sy, fy);
    }
    energy[(size_t)j * HW + p] = v;
  }
}

}  // namespace ups

extern "C" int upsnet_mask_removal(const float* boxes, const float* cls_prob, const float* mask_logit,
                                   const int64_t* cls_idx, int n, const int* n_dev, int H, int W, int num_thing,
                                   double fraction_threshold, int64_t* keep_out, int* k_out, float* mask_energy,
                                   void* workspace, size_t workspace_bytes, void* stream) {
  using namespace ups;
  if (!boxes || !cls_prob || !mask_logit || !cls_idx || !keep_out || !k_out || !workspace) return UPSNET_E_BADARG;
  if (n < 1 || H <= 0 || W <= 0 || num_thing <= 0) return UPSNET_E_BADARG;
  if (n > kMaxList) return UPSNET_E_UNSUPPORTED;
  PanWorkspace ws;
  const size_t need = pan_ws_layout(n, H, W, num_thing, ws, workspace, workspace_bytes);
  if (need == 0 || workspace_bytes < need) return UPSNET_E_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const int Ww = ceil_div(W, 32);
  UPS_CUDA(cudaMemsetAsync(ws.occ, 0, (size_t)num_thing * H * Ww * sizeof(unsigned int), st));
  UPS_CUDA(cudaMemsetAsync(ws.kept_flag, 0, sizeof(int) * n, st));
  pan_prep_kernel<<<1, kPrepThreads, 0, st>>>(boxes, cls_prob, cls_idx, n, n_dev, H, W, ws);
  UPS_CHECK_LAUNCH();
  {
    static ups::PerDeviceOnce configured;
    if (configured.need()) {   // up to kMaxList * 32 B of per-instance metadata
      UPS_CUDA(cudaFuncSetAttribute(pan_decide_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxList * 32));
    }
  }
  for (int rq = 0; rq < ws.rounds; ++rq) {   // one round unless n * H * W/32 words exceed the bit-window budget
    pan_bits_kernel<<<dim3(kBitsChunks, n), kBitsThreads, 0, st>>>(mask_logit, n, n_dev, rq, ws);
    UPS_CHECK_LAUNCH();
    pan_decide_kernel<<<num_thing, kDecideThreads, (size_t)n * 32, st>>>(n, n_dev, H, W, fraction_threshold, rq, ws);
    UPS_CHECK_LAUNCH();
  }
  pan_compact_kernel<<<1, kCompactThreads, 0, st>>>(n, n_dev, ws, keep_out, k_out);
  UPS_CHECK_LAUNCH();
  if (mask_energy) {
    dim3 grid((unsigned)min((size_t)kNumSMs * 8, ((size_t)H * W + 255) / 256), (unsigned)n);
    pan_paste_kernel<<<grid, 256, 0, st>>>(mask_logit, H, W, ws, mask_energy);
    UPS_CHECK_LAUNCH();
  }
  return 0;
}

extern "C" int upsnet_panoptic_workspace_bytes(int n, int H, int W, int num_thing, size_t* bytes) {
  if (!bytes || n < 0 || H <= 0 || W <= 0 || num_thing <= 0) return UPSNET_E_BADARG;
  ups::PanWorkspace ws;
  *bytes = ups::pan_ws_layout(n, H, W, num_thing, ws, nullptr);
  return 0;
}

extern "C" int upsnet_panoptic_workspace_min_bytes(int n, int H, int W, int num_thing, size_t* bytes) {
  if (!bytes || n < 0 || H <= 0 || W <= 0 || num_thing <= 0) return UPSNET_E_BADARG;
  // fixed part + the smallest bit-window budget: max(one window, all windows / kMaxRounds), plus the spill window
  ups::PanWorkspace ws;
  const size_t full = ups::pan_ws_layout(n, H, W, num_thing, ws, nullptr);
  const long long win = (long long)H * ups::ceil_div(W, 32), all = win * (n > 0 ? n : 1);
  long long budget = all < ups::kBitsBudget ? all : ups::kBitsBudget;
  long long minb = (all + ups::kMaxRounds - 1) / ups::kMaxRounds;
  if (minb < win) minb = win;
  *bytes = full - (size_t)(budget - minb) * sizeof(unsigned int) + 1024;
  return 0;
}

static int panoptic_head_impl(const float* fcn, bool up4, int S, int H, int W, const float* boxes,
                              const float* cls_prob, const float* mask_logit,
                              const int64_t* cls_idx, int n, const int* n_dev, int num_stuff,
                              double fraction_threshold, int64_t* keep_out, int* k_out,
                              int64_t* labels, int64_t* sem_labels, void* workspace,
                              size_t workspace_bytes, void* stream) {
  using namespace ups;
  if (!fcn || !boxes || !cls_prob || !mask_logit || !cls_idx || !keep_out || !k_out || !labels || !workspace)
    return UPSNET_E_BADARG;
  const int num_thing = S - num_stuff;
  if (n < 1 || H <= 0 || W <= 0 || num_thing <= 0 || num_stuff < 1) return UPSNET_E_BADARG;
  if (n > kMaxList) return UPSNET_E_UNSUPPORTED;  // per-tile instance list capacity
  if (((uintptr_t)fcn & 15) || ((uintptr_t)labels & 15) || (sem_labels && ((uintptr_t)sem_labels & 15)))
    return UPSNET_E_BADARG;
  PanWorkspace ws;
  const size_t need = pan_ws_layout(n, H, W, num_thing, ws, workspace, workspace_bytes);
  if (need == 0 || workspace_bytes < need) return UPSNET_E_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const int Ww = ceil_div(W, 32);
  UPS_CUDA(cudaMemsetAsync(ws.occ, 0, (size_t)num_thing * H * Ww * sizeof(unsigned int), st));
  UPS_CUDA(cudaMemsetAsync(ws.kept_flag, 0, sizeof(int) * n, st));
  pan_prep_kernel<<<1, kPrepThreads, 0, st>>>(boxes, cls_prob, cls_idx, n, n_dev, H, W, ws);
  UPS_CHECK_LAUNCH();
  {
    static ups::PerDeviceOnce configured;
    if (configured.need()) {   // up to kMaxList * 32 B of per-instance metadata
      UPS_CUDA(cudaFuncSetAttribute(pan_decide_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxList * 32));
    }
  }
  for (int rq = 0; rq < ws.rounds; ++rq) {   // one round unless n * H * W/32 words exceed the bit-window budget
    pan_bits_kernel<<<dim3(kBitsChunks, n), kBitsThreads, 0, st>>>(mask_logit, n, n_dev, rq, ws);
    UPS_CHECK_LAUNCH();
    pan_decide_kernel<<<num_thing, kDecideThreads, (size_t)n * 32, st>>>(n, n_dev, H, W, fraction_threshold, rq, ws);
    UPS_CHECK_LAUNCH();
  }
  pan_compact_kernel<<<1, kCompactThreads, 0, st>>>(n, n_dev, ws, keep_out, k_out);
  UPS_CHECK_LAUNCH();
  dim3 grid(ceil_div(W, kTileW), ceil_div(H, kTileH));
  if (up4) pan_fuse_kernel<true><<<grid, kFuseThreads, 0, st>>>(fcn, S, H, W, num_stuff, mask_logit, ws, labels, sem_labels);
  else pan_fuse_kernel<false><<<grid, kFuseThreads, 0, st>>>(fcn, S, H, W, num_stuff, mask_logit, ws, labels, sem_labels);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_panoptic_head(const float* fcn, int S, int H, int W, const float* boxes,
                                    const float* cls_prob, const float* mask_logit,
                                    const int64_t* cls_idx, int n, const int* n_dev, int num_stuff,
                                    double fraction_threshold, int64_t* keep_out, int* k_out,
                                    int64_t* labels, int64_t* sem_labels, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  return panoptic_head_impl(fcn, false, S, H, W, boxes, cls_prob, mask_logit, cls_idx, n, n_dev, num_stuff, fraction_threshold,
                            keep_out, k_out, labels, sem_labels, workspace, workspace_bytes, stream);
}

extern "C" int upsnet_panoptic_head_up4(const float* score, int S, int Hs, int Ws, const float* boxes,
                                        const float* cls_prob, const float* mask_logit,
                                        const int64_t* cls_idx, int n, const int* n_dev, int num_stuff,
                                        double fraction_threshold, int64_t* keep_out, int* k_out,
                                        int64_t* labels, int64_t* sem_labels, void* workspace,
                                        size_t workspace_bytes, void* stream) {
  if (Hs <= 0 || Ws <= 0 || Hs > (1 << 28) || Ws > (1 << 28)) return UPSNET_E_BADARG;
  return panoptic_head_impl(score, true, S, 4 * Hs, 4 * Ws, boxes, cls_prob, mask_logit, cls_idx, n, n_dev, num_stuff,
                            fraction_threshold, keep_out, k_out, labels, sem_labels, workspace, workspace_bytes, stream);
}
