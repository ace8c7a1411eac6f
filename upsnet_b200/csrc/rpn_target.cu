// rpn_target.cu -- RPN training targets of one image (rpn/assign_anchor.py:447-595 _get_rpn_blobs, called by
// add_rpn_blobs from the training data loaders), replacing the host's float32 IoU matrix of every inside anchor against
// every ground-truth box, its argmaxes and tie sets, the two np.random.choice draws and the dense per-level arrays.
//
// Launches (none synchronises the host; every count stays on the device):
//   1. rt_max:     per anchor: inside test, IoU against every box (boxes staged through shared memory in chunks),
//                  max and first argmax; per box: max over the inside anchors (atomicMax on the bit pattern, IoU >= 0)
//   2. rt_label:   per anchor: fg candidate (IoU == some box's max, or max >= pos), bg candidate (max < neg); per-CTA counts
//   3. rt_scan:    CTA offsets, totals, and what each draw has to do
//   4. rt_compact: candidate lists in anchor order with the 64-bit key of each position (the seeded rule of np.random.choice)
//   5. rt_select:  8 radix passes: the exact k-th smallest key of each draw
//   6. rt_mark:    the drawn anchors (<= batch of them) into two short lists
//   7. rt_write:   one CTA writes labels, box targets and weights of those anchors over the constant fill
#include "anchors.cuh"
#include "common.cuh"
#include "cta.cuh"
#include "targets.cuh"

namespace ups {

constexpr int kRtThreads = 256;     // anchors per CTA in the per-anchor passes
constexpr int kRtChunk = 1024;      // boxes staged in shared memory at a time
constexpr int kRtMaxG = UPSNET_RPN_TARGETS_MAX_G;
constexpr int kRtLevels = 8;
constexpr int kRtSelBlocks = 264;   // grid-stride CTAs of the select / mark passes, per draw

enum { kFlagInside = 1, kFlagFg = 2, kFlagBg = 4, kFlagBgDrawn = 8 };
enum { kDrawAll = 0, kDrawNone = 1, kDrawSelect = 2 };

struct RtState {
  unsigned int hist[2][256];
  unsigned long long prefix[2];     // after the 8 passes: the k-th smallest key of the draw
  int n[2], k[2], need[2], mode[2];
  unsigned int ticket[2];
  int list_cnt[2];
};

struct RtParams {
  const float* gt;                  // [G,4]
  const double* cell;               // [L,A,4]
  long long off[kRtLevels + 1];     // first anchor of each level
  int F[kRtLevels], stride[kRtLevels];
  int L, A, N, G, nblk, batch, num_fg;
  double im_h, im_w, straddle;
  float pos, neg;
  unsigned long long seed;
  // workspace
  RtState* st;
  unsigned int* gtmax;              // [G] float bits
  float* amax;                      // [N]
  int* aarg;                        // [N]
  unsigned char* flags;             // [N]
  int* blk;                         // [nblk][3] fg, bg, inside counts; then [nblk][2] fg, bg offsets
  unsigned long long* keys[2];      // [N] per draw, in candidate order
  int* idx[2];                      // [N] anchor of each candidate
  int* list[2];                     // [batch] drawn anchors
  // outputs
  int64_t* labels;
  float *targets, *inside_w, *outside_w;
  int* counts;
};

__device__ __forceinline__ int anchor_level(const RtParams& p, int n) {
  int l = 0;
  while (l + 1 < p.L && n >= p.off[l + 1]) ++l;
  return l;
}

// where anchor n (the reference's order: level, then cell (y, x), then a) lives in the per-level blobs
struct AnchorPos {
  int l, a, yx, FF;
  float4 box;
};

__device__ __forceinline__ AnchorPos anchor_of(const RtParams& p, int n) {
  AnchorPos o;
  o.l = anchor_level(p, n);
  const int r = n - (int)p.off[o.l];
  const int cell = r / p.A;
  o.a = r - cell * p.A;
  const int F = p.F[o.l], y = cell / F, x = cell - y * F;
  o.yx = y * F + x;
  o.FF = F * F;
  o.box = shifted_anchor(p.cell + ((size_t)o.l * p.A + o.a) * 4, x, y, p.stride[o.l]);
  return o;
}

// element of the labels blob [1,A,F,F] and first element of the [1,4A,F,F] blobs (channel a*4 + c), levels concatenated
__device__ __forceinline__ size_t label_at(const RtParams& p, const AnchorPos& q) {
  return (size_t)p.off[q.l] + (size_t)q.a * q.FF + q.yx;
}
__device__ __forceinline__ size_t coord_at(const RtParams& p, const AnchorPos& q) {
  return 4 * (size_t)p.off[q.l] + (size_t)(4 * q.a) * q.FF + q.yx;
}

__device__ __forceinline__ bool is_inside(const RtParams& p, float4 an) {
  if (p.straddle < 0.0) return true;
  return (double)an.x >= -p.straddle && (double)an.y >= -p.straddle && (double)an.z < p.im_w + p.straddle &&
         (double)an.w < p.im_h + p.straddle;
}

__device__ __forceinline__ float4 load_box(const float* gt, int k) {
  return make_float4(__ldg(gt + 4 * k), __ldg(gt + 4 * k + 1), __ldg(gt + 4 * k + 2), __ldg(gt + 4 * k + 3));
}

// 1. per-anchor max / first argmax and per-box max
__global__ void __launch_bounds__(kRtThreads) rt_max_kernel(const RtParams p) {
  __shared__ float4 sbox[kRtChunk];
  __shared__ float sarea[kRtChunk];
  __shared__ unsigned int smax[kRtChunk];
  const int n = blockIdx.x * kRtThreads + threadIdx.x;
  bool inside = false;
  float4 an = make_float4(0.f, 0.f, 0.f, 0.f);
  if (n < p.N) {
    an = anchor_of(p, n).box;
    inside = is_inside(p, an);
  }
  const double a_area = area64(an);
  float best = -1.f;
  int arg = 0;
  for (int c0 = 0; c0 < p.G; c0 += kRtChunk) {
    const int cn = min(kRtChunk, p.G - c0);
    __syncthreads();
    for (int k = threadIdx.x; k < cn; k += kRtThreads) {
      const float4 q = load_box(p.gt, c0 + k);
      sbox[k] = q;
      sarea[k] = (float)area64(q);
      smax[k] = 0u;
    }
    __syncthreads();
    if (inside) {
      for (int k = 0; k < cn; ++k) {
        const float o = pair_iou(an, a_area, sbox[k], sarea[k]);
        if (o > best) { best = o; arg = c0 + k; }     // strict: the first argmax, as numpy's
        const unsigned int b = __float_as_uint(o);
        if (b > smax[k]) atomicMax(&smax[k], b);
      }
    }
    __syncthreads();
    for (int k = threadIdx.x; k < cn; k += kRtThreads)
      if (smax[k]) atomicMax(&p.gtmax[c0 + k], smax[k]);
  }
  if (n < p.N) {
    p.amax[n] = best;
    p.aarg[n] = arg;
    p.flags[n] = inside ? kFlagInside : 0;
  }
}

// 2. candidate flags; an anchor is fg when one of its IoUs equals that box's max (boxes whose max is 0 included)
__global__ void __launch_bounds__(kRtThreads) rt_label_kernel(const RtParams p) {
  __shared__ float4 sbox[kRtChunk];
  __shared__ float sarea[kRtChunk];
  __shared__ float smax[kRtChunk];
  const int n = blockIdx.x * kRtThreads + threadIdx.x;
  bool inside = false, fg = false, bg = false;
  float4 an = make_float4(0.f, 0.f, 0.f, 0.f);
  if (n < p.N) {
    inside = (p.flags[n] & kFlagInside) != 0;
    if (inside) {
      const float m = p.amax[n];
      fg = m >= p.pos;
      bg = m < p.neg;
      an = anchor_of(p, n).box;
    }
  }
  const double a_area = area64(an);
  bool look = inside && !fg;
  for (int c0 = 0; c0 < p.G; c0 += kRtChunk) {
    const int cn = min(kRtChunk, p.G - c0);
    __syncthreads();
    for (int k = threadIdx.x; k < cn; k += kRtThreads) {
      const float4 q = load_box(p.gt, c0 + k);
      sbox[k] = q;
      sarea[k] = (float)area64(q);
      smax[k] = __uint_as_float(__ldcg(p.gtmax + c0 + k));
    }
    __syncthreads();
    if (look) {
      for (int k = 0; k < cn; ++k)
        if (pair_iou(an, a_area, sbox[k], sarea[k]) == smax[k]) { fg = true; look = false; break; }
    }
  }
  if (n < p.N) p.flags[n] = (inside ? kFlagInside : 0) | (fg ? kFlagFg : 0) | (bg ? kFlagBg : 0);
  const int cf = __syncthreads_count(fg), cb = __syncthreads_count(bg), ci = __syncthreads_count(inside);
  if (threadIdx.x == 0) {
    p.blk[3 * blockIdx.x] = cf;
    p.blk[3 * blockIdx.x + 1] = cb;
    p.blk[3 * blockIdx.x + 2] = ci;
  }
}

// 3. CTA offsets of both candidate lists and the plan of both draws (one CTA)
constexpr int kRtScanThreads = 1024;

__global__ void __launch_bounds__(kRtScanThreads) rt_scan_kernel(const RtParams p) {
  __shared__ int warp_sums[kRtScanThreads / 32];
  int carry_f = 0, carry_b = 0, carry_i = 0;
  int* off = p.blk + 3 * p.nblk;
  for (int b0 = 0; b0 < p.nblk; b0 += kRtScanThreads) {
    const int b = b0 + threadIdx.x;
    const bool ok = b < p.nblk;
    int tf, tb, ti;
    const int ef = cta_scan_excl<kRtScanThreads>(ok ? p.blk[3 * b] : 0, warp_sums, &tf);
    const int eb = cta_scan_excl<kRtScanThreads>(ok ? p.blk[3 * b + 1] : 0, warp_sums, &tb);
    cta_scan_excl<kRtScanThreads>(ok ? p.blk[3 * b + 2] : 0, warp_sums, &ti);
    if (ok) { off[2 * b] = carry_f + ef; off[2 * b + 1] = carry_b + eb; }
    carry_f += tf; carry_b += tb; carry_i += ti;
  }
  if (threadIdx.x == 0) {
    RtState* st = p.st;
    const int nf = carry_f, nb = carry_b;
    p.counts[0] = carry_i;
    p.counts[1] = nf;
    // fg: when nf > num_fg, np.random.choice disables the nf - num_fg smallest keys, i.e. keeps the num_fg largest
    st->n[0] = nf;
    st->mode[0] = nf > p.num_fg ? kDrawSelect : kDrawAll;
    st->k[0] = st->need[0] = p.num_fg;
    // bg: num_bg = batch - #(label 1); with no more candidates than that, no anchor is labelled 0
    const int num_bg = p.batch - min(nf, p.num_fg);
    st->n[1] = nb;
    st->mode[1] = (nb > num_bg && num_bg > 0) ? kDrawSelect : kDrawNone;
    st->k[1] = st->need[1] = num_bg;
  }
}

// 4. candidate lists in anchor order (= the reference's index lists) with the key of each position:
//    key(s, pos) = splitmix64(s ^ pos * golden gamma), s = seed (fg) or splitmix64(seed) (bg); fg keys are stored inverted so
//    that both draws select the k smallest
__global__ void __launch_bounds__(kRtThreads) rt_compact_kernel(const RtParams p) {
  __shared__ int warp_n[kRtThreads / 32];
  const int n = blockIdx.x * kRtThreads + threadIdx.x;
  const int fl = n < p.N ? p.flags[n] : 0;
  const bool fg = fl & kFlagFg, bg = fl & kFlagBg;
  int tot;
  const int rf = cta_ballot_rank<kRtThreads>(fg, warp_n, &tot), rb = cta_ballot_rank<kRtThreads>(bg, warp_n, &tot);
  const int* off = p.blk + 3 * p.nblk + 2 * blockIdx.x;
  if (fg) {
    const int pos = off[0] + rf;
    p.keys[0][pos] = ~draw_key(p.seed, 0, (unsigned long long)pos);
    p.idx[0][pos] = n;
  }
  if (bg) {
    const int pos = off[1] + rb;
    p.keys[1][pos] = draw_key(p.seed, 1, (unsigned long long)pos);
    p.idx[1][pos] = n;
  }
}

// 5. one 8-bit digit of the radix select of both draws (blockIdx.y); the last CTA of a draw fixes the digit
__global__ void __launch_bounds__(kRtThreads) rt_select_kernel(const RtParams p, int shift) {
  const int s = blockIdx.y;
  RtState* st = p.st;
  if (st->mode[s] != kDrawSelect) return;
  __shared__ unsigned int sh[256];
  sh[threadIdx.x] = 0u;
  __syncthreads();
  const int n = st->n[s];
  const unsigned long long prefix = st->prefix[s];
  const unsigned long long mask_hi = shift >= 56 ? 0ull : (~0ull << (shift + 8));
  const unsigned long long* keys = p.keys[s];
  for (int i = blockIdx.x * kRtThreads + threadIdx.x; i < n; i += gridDim.x * kRtThreads) {
    const unsigned long long key = keys[i];
    if ((key & mask_hi) == prefix) atomicAdd(&sh[(unsigned)(key >> shift) & 255u], 1u);
  }
  __syncthreads();
  if (sh[threadIdx.x]) atomicAdd(&st->hist[s][threadIdx.x], sh[threadIdx.x]);
  if (!last_cta(&st->ticket[s], gridDim.x)) return;
  sh[threadIdx.x] = __ldcg(&st->hist[s][threadIdx.x]);
  st->hist[s][threadIdx.x] = 0u;
  __syncthreads();
  RadixDigit d;
  if (threadIdx.x < 32 && warp_radix_digit<256, false>(sh, st->need[s], &d)) {
    st->need[s] = d.need;
    st->prefix[s] = prefix | ((unsigned long long)d.digit << shift);
    st->ticket[s] = 0u;
  }
}

// 6. the drawn anchors: fg keeps (keys <= the k-th), bg labels them 0 and flags them for rt_write
__global__ void __launch_bounds__(kRtThreads) rt_mark_kernel(const RtParams p) {
  const int s = blockIdx.y;
  RtState* st = p.st;
  const int mode = st->mode[s];
  if (mode == kDrawNone) return;
  const int n = st->n[s];
  const unsigned long long kth = st->prefix[s];
  for (int i = blockIdx.x * kRtThreads + threadIdx.x; i < n; i += gridDim.x * kRtThreads) {
    if (mode == kDrawAll || p.keys[s][i] <= kth) {
      const int a = p.idx[s][i];
      p.list[s][atomicAdd(&st->list_cnt[s], 1)] = a;
      if (s == 1) p.flags[a] |= kFlagBgDrawn;
    }
  }
}

// 7. the drawn anchors over the constant fill (labels -1, everything else 0); one CTA
__global__ void __launch_bounds__(kRtThreads) rt_write_kernel(const RtParams p) {
  RtState* st = p.st;
  const int nfs = st->list_cnt[0], nbs = st->list_cnt[1];
  int overlap = 0;     // fg-stage anchors relabelled 0 by the bg draw
  for (int i0 = 0; i0 < nfs; i0 += kRtThreads) {
    const int i = i0 + threadIdx.x;
    overlap += __syncthreads_count(i < nfs && (p.flags[p.list[0][i]] & kFlagBgDrawn));
  }
  const int num_examples = nfs + nbs - overlap;
  const float w = num_examples > 0 ? (float)__ddiv_rn(1.0, (double)num_examples) : 0.f;
  for (int i = threadIdx.x; i < nbs; i += kRtThreads) {
    const AnchorPos q = anchor_of(p, p.list[1][i]);
    p.labels[label_at(p, q)] = 0;
    float* ow = p.outside_w + coord_at(p, q);
    for (int c = 0; c < 4; ++c) ow[(size_t)c * q.FF] = w;
  }
  for (int i = threadIdx.x; i < nfs; i += kRtThreads) {
    const int n = p.list[0][i];
    const AnchorPos q = anchor_of(p, n);
    const size_t base = coord_at(p, q);
    const float4 t = box_target(q.box, load_box(p.gt, p.aarg[n]), make_float4(1.f, 1.f, 1.f, 1.f));
    p.targets[base] = t.x;
    p.targets[base + q.FF] = t.y;
    p.targets[base + 2 * (size_t)q.FF] = t.z;
    p.targets[base + 3 * (size_t)q.FF] = t.w;
    if (!(p.flags[n] & kFlagBgDrawn)) {
      p.labels[label_at(p, q)] = 1;
      for (int c = 0; c < 4; ++c) {
        p.inside_w[base + (size_t)c * q.FF] = 1.f;
        p.outside_w[base + (size_t)c * q.FF] = w;
      }
    }
  }
  if (threadIdx.x == 0) {
    p.counts[2] = nfs - overlap;
    p.counts[3] = nbs;
  }
}

inline size_t rt_layout(long long N, int batch, void* base, RtParams& p) {
  const long long nblk = (N + kRtThreads - 1) / kRtThreads;
  WsCarve c(base);
  p.st = c.take<RtState>(1);
  p.gtmax = c.take<unsigned int>(kRtMaxG);
  p.amax = c.take<float>(N);
  p.aarg = c.take<int>(N);
  p.flags = c.take<unsigned char>(N);
  p.blk = c.take<int>(nblk * 5);
  p.keys[0] = c.take<unsigned long long>(N);
  p.keys[1] = c.take<unsigned long long>(N);
  p.idx[0] = c.take<int>(N);
  p.idx[1] = c.take<int>(N);
  p.list[0] = c.take<int>(batch);
  p.list[1] = c.take<int>(batch);
  return c.bytes();
}

}  // namespace ups

extern "C" int upsnet_rpn_targets_workspace_bytes(long long num_anchors, int batch_size, size_t* bytes) {
  if (!bytes || num_anchors <= 0 || num_anchors >= (1ll << 31) || batch_size <= 0) return UPSNET_E_BADARG;
  ups::RtParams p{};
  *bytes = ups::rt_layout(num_anchors, batch_size, nullptr, p);
  return 0;
}

extern "C" int upsnet_rpn_targets(const float* gt_boxes, int G, const double* cell_anchors, const int* strides,
                                  const int* field_sizes, int L, int A, double im_height, double im_width,
                                  double straddle_thresh, float positive_overlap, float negative_overlap, int batch_size,
                                  int num_fg, unsigned long long seed, int64_t* labels, float* bbox_targets,
                                  float* inside_weights, float* outside_weights, int* counts, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  using namespace ups;
  if (!gt_boxes || !cell_anchors || !strides || !field_sizes || !labels || !bbox_targets || !inside_weights ||
      !outside_weights || !counts || !workspace)
    return UPSNET_E_BADARG;
  if (G <= 0 || L <= 0 || L > kRtLevels || A <= 0 || batch_size <= 0 || num_fg <= 0 || num_fg > batch_size)
    return UPSNET_E_BADARG;
  if (G > kRtMaxG) return UPSNET_E_UNSUPPORTED;
  RtParams p{};
  long long N = 0;
  for (int l = 0; l < L; ++l) {
    if (field_sizes[l] <= 0 || strides[l] <= 0) return UPSNET_E_BADARG;
    p.off[l] = N;
    p.F[l] = field_sizes[l];
    p.stride[l] = strides[l];
    N += (long long)A * field_sizes[l] * field_sizes[l];
  }
  p.off[L] = N;
  if (N >= (1ll << 31)) return UPSNET_E_UNSUPPORTED;
  if (workspace_bytes < rt_layout(N, batch_size, workspace, p)) return UPSNET_E_WORKSPACE;
  p.gt = gt_boxes; p.cell = cell_anchors;
  p.L = L; p.A = A; p.N = (int)N; p.G = G; p.nblk = (int)((N + kRtThreads - 1) / kRtThreads);
  p.batch = batch_size; p.num_fg = num_fg;
  p.im_h = im_height; p.im_w = im_width; p.straddle = straddle_thresh;
  p.pos = positive_overlap; p.neg = negative_overlap; p.seed = seed;
  p.labels = labels; p.targets = bbox_targets; p.inside_w = inside_weights; p.outside_w = outside_weights;
  p.counts = counts;
  cudaStream_t st = (cudaStream_t)stream;
  UPS_CUDA(cudaMemsetAsync(p.st, 0, sizeof(RtState), st));
  UPS_CUDA(cudaMemsetAsync(p.gtmax, 0, (size_t)G * 4, st));
  // the constant fill of the outputs: label -1 (all bytes 0xff), targets and weights 0
  UPS_CUDA(cudaMemsetAsync(labels, 0xff, (size_t)N * 8, st));
  UPS_CUDA(cudaMemsetAsync(bbox_targets, 0, (size_t)N * 16, st));
  UPS_CUDA(cudaMemsetAsync(inside_weights, 0, (size_t)N * 16, st));
  UPS_CUDA(cudaMemsetAsync(outside_weights, 0, (size_t)N * 16, st));
  rt_max_kernel<<<p.nblk, kRtThreads, 0, st>>>(p);
  UPS_CHECK_LAUNCH();
  rt_label_kernel<<<p.nblk, kRtThreads, 0, st>>>(p);
  UPS_CHECK_LAUNCH();
  rt_scan_kernel<<<1, kRtScanThreads, 0, st>>>(p);
  UPS_CHECK_LAUNCH();
  rt_compact_kernel<<<p.nblk, kRtThreads, 0, st>>>(p);
  UPS_CHECK_LAUNCH();
  for (int shift = 56; shift >= 0; shift -= 8) {
    rt_select_kernel<<<dim3(kRtSelBlocks, 2), kRtThreads, 0, st>>>(p, shift);
    UPS_CHECK_LAUNCH();
  }
  rt_mark_kernel<<<dim3(kRtSelBlocks, 2), kRtThreads, 0, st>>>(p);
  UPS_CHECK_LAUNCH();
  rt_write_kernel<<<1, kRtThreads, 0, st>>>(p);
  UPS_CHECK_LAUNCH();
  return 0;
}
