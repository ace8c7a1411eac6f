// panoptic_loss.cu -- the panoptic head of the TRAINING forward (models/resnet_upsnet.py:156-179, 250-257) as one fused
// loss: SegTerm + MaskTerm + void logits + MaskMatching + cross-entropy + accuracy, forward and backward, evaluated per
// pixel over a small instance table.  No [1,k,h,w] plane exists in global memory; backward needs 8 bytes per pixel (the
// log-sum-exp and the ground-truth channel).  See include/upsnet_b200.h for the contract of every symbol.
//
// Determinism: every output element has one owner thread that sums in a fixed order, the loss and the counts go through
// per-block partials and a fixed-order second stage; there is no atomic in this file.
#include "common.cuh"
#include "cta.cuh"
#include "targets.cuh"

namespace ups {
namespace {

constexpr int kPlThreads = 256;
constexpr int kPlMaxM = 32;                 // one source column per lane in pl_mask_grad_kernel
constexpr size_t kPlSmemTable = 40 * 1024;  // larger instance tables are read from global memory
constexpr int kPlInvalid = -1;              // a label that is neither a channel nor 255: no loss, no gradient

struct PlInst {
  int sx0, sy0, sx1, sy1;  // SegTerm window [x0,x1) x [y0,y1), clamped to the image; empty when the class is 0
  int mx0, my0;            // MaskTerm paste origin (r0, r1); may lie left of / above the image
  int bw, bh;              // size the M x M logit is resized to
  int ex, ey;              // MaskTerm window end (exclusive), min(r2 + 1, w) / min(r3 + 1, h)
  float scx, scy;          // ATen's area_pixel scale M / bw, M / bh (float32)
  int tch;                 // seg channel of the instance's class, -1 when SegTerm skips it
  int moff;                // element offset of the instance's M x M logit in mask_score
};

struct PlArgs {
  const float* fcn; const float* mask; const float* rois; const int64_t* cls;
  const int64_t* seg_gt; const void* mask_gt; const int64_t* keep;
  PlInst* tab;
  int S, h, w, k, C, M, G, num_classes, num_stuff, enable_void, tab_smem;
  float box_scale;
  // forward outputs / backward inputs
  float* lse; int* gtc; double* part_loss; int* part_cnt;
  const float* grad_out; float* dfcn; float* dmask;
};

// float -> int as Python's int() / Tensor.long() do (truncation toward zero), saturated so the cast is defined
__device__ __forceinline__ int pl_trunc(float v) { return (int)fminf(fmaxf(v, -1.0e9f), 1.0e9f); }

__global__ void pl_table_kernel(PlArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.k) return;
  const float b0 = __fmul_rn(a.rois[i * 5 + 1], a.box_scale), b1 = __fmul_rn(a.rois[i * 5 + 2], a.box_scale);
  const float b2 = __fmul_rn(a.rois[i * 5 + 3], a.box_scale), b3 = __fmul_rn(a.rois[i * 5 + 4], a.box_scale);
  long long c = a.cls[i];
  if (c < 0 || c >= a.num_classes) c = 0;
  PlInst t;
  // unary_logits.py:99-103: int() of the near corner, int(round half to even + 1) of the far one, slice clamping
  t.sx0 = min(max(pl_trunc(b0), 0), a.w);
  t.sy0 = min(max(pl_trunc(b1), 0), a.h);
  t.sx1 = min(max(pl_trunc(__fadd_rn(rintf(b2), 1.f)), 0), a.w);
  t.sy1 = min(max(pl_trunc(__fadd_rn(rintf(b3), 1.f)), 0), a.h);
  t.tch = c > 0 ? a.num_stuff + (int)c - 1 : -1;
  if (c == 0) t.sx1 = t.sx0, t.sy1 = t.sy0;
  // unary_logits.py:54-63: .long() of all four corners
  const int r0 = pl_trunc(b0), r1 = pl_trunc(b1), r2 = pl_trunc(b2), r3 = pl_trunc(b3);
  t.mx0 = r0; t.my0 = r1;
  t.bw = max(r2 - r0 + 1, 1); t.bh = max(r3 - r1 + 1, 1);
  t.ex = min(r2 + 1, a.w); t.ey = min(r3 + 1, a.h);
  t.scx = __fdiv_rn((float)a.M, (float)t.bw); t.scy = __fdiv_rn((float)a.M, (float)t.bh);
  t.moff = (i * a.C + (a.C == 1 ? 0 : (int)c)) * a.M * a.M;
  a.tab[i] = t;
}

// ATen's bilinear source index for align_corners = False: max(scale * (dst + 0.5) - 0.5, 0), each operation rounded
__device__ __forceinline__ float pl_src(int d, float scale) {
  return fmaxf(__fsub_rn(__fmul_rn(scale, __fadd_rn((float)d, 0.5f)), 0.5f), 0.f);
}
__device__ __forceinline__ int pl_i0(int d, float scale, int M) { return min((int)pl_src(d, scale), M - 1); }

struct PlTap { int i0, i1; float l0, l1; };
__device__ __forceinline__ PlTap pl_tap(int d, float scale, int M) {
  const float s = pl_src(d, scale);
  PlTap t;
  t.i0 = min((int)s, M - 1);
  t.i1 = t.i0 + (t.i0 < M - 1 ? 1 : 0);
  t.l1 = __fsub_rn(s, (float)t.i0);
  t.l0 = __fsub_rn(1.f, t.l1);
  return t;
}

__device__ __forceinline__ float pl_mask_value(const float* __restrict__ m, int M, const PlTap& ty, const PlTap& tx) {
  const float* r0 = m + ty.i0 * M;
  const float* r1 = m + ty.i1 * M;
  const float a = __fmaf_rn(tx.l1, __ldg(r0 + tx.i1), __fmul_rn(tx.l0, __ldg(r0 + tx.i0)));
  const float b = __fmaf_rn(tx.l1, __ldg(r1 + tx.i1), __fmul_rn(tx.l0, __ldg(r1 + tx.i0)));
  return __fmaf_rn(ty.l1, b, __fmul_rn(ty.l0, a));
}

// the two terms of instance channel t at pixel (y, x) = p: (SegTerm value, whether its window covers p, MaskTerm value)
__device__ __forceinline__ void pl_inst_terms(const PlInst& t, const PlArgs& a, int p, int y, int x, float* seg, bool* cov,
                                              float* msk) {
  *cov = x >= t.sx0 && x < t.sx1 && y >= t.sy0 && y < t.sy1;
  *seg = *cov ? __ldg(a.fcn + (size_t)t.tch * a.h * a.w + p) : 0.f;
  *msk = 0.f;
  if (x >= t.mx0 && x < t.ex && y >= t.my0 && y < t.ey)
    *msk = pl_mask_value(a.mask + t.moff, a.M, pl_tap(y - t.my0, t.scy, a.M), pl_tap(x - t.mx0, t.scx, a.M));
}

// mask_matching.py:45-56 at one pixel, as the int64 value the reference writes
template <typename MT>
__device__ __forceinline__ long long pl_gt_value(const int64_t* seg_gt, const MT* mask_gt, const int64_t* keep, int n, int G,
                                                 int hw, int p, int num_stuff) {
  const long long s = seg_gt[p];
  long long g = (s <= num_stuff - 1 || s >= 255) ? s : -1;
  for (int j = n - 1; j >= 0; --j) {          // later instances overwrite earlier ones: the last hit wins
    const long long gi = keep ? keep[j] : j;
    if (gi < 0 || gi >= G) continue;
    const MT m = mask_gt[(size_t)gi * hw + p];
    if (m != 0 && m != 255) { g = num_stuff + j; break; }
  }
  if (g == -1) g = keep ? num_stuff + n : 255;
  return g;
}

__device__ __forceinline__ const PlInst* pl_stage_table(const PlArgs& a, PlInst* s_tab) {
  if (!a.tab_smem) return a.tab;
  const int n = a.k * (int)(sizeof(PlInst) / 4);
  for (int j = threadIdx.x; j < n; j += blockDim.x) ((int*)s_tab)[j] = ((const int*)a.tab)[j];
  __syncthreads();
  return s_tab;
}

template <typename MT>
__global__ void __launch_bounds__(kPlThreads) pl_forward_kernel(PlArgs a) {
  extern __shared__ PlInst s_tab[];
  const PlInst* tab = pl_stage_table(a, s_tab);
  const int hw = a.h * a.w, p = blockIdx.x * kPlThreads + threadIdx.x;
  const int nch = a.num_stuff + a.k + (a.enable_void ? 1 : 0);
  double loss[1] = {0.0};
  int cnt[2] = {0, 0};              // correct, ignored
  if (p < hw) {
    const int y = p / a.w, x = p - y * a.w;
    const long long g = pl_gt_value<MT>(a.seg_gt, (const MT*)a.mask_gt, a.keep, a.keep ? a.k : a.G, a.G, hw, p, a.num_stuff);
    // streaming log-sum-exp over the channels in their order; the first maximum is the arg-max (ties: lowest channel)
    float m = -INFINITY, s = 0.f, lg = 0.f;
    int am = 0;
    auto push = [&](int c, float v) {
      if (v > m) { s = __fmaf_rn(s, expf(m - v), 1.f); m = v; am = c; }
      else s += expf(v - m);
      if (c == g) lg = v;
    };
    for (int c = 0; c < a.num_stuff; ++c) push(c, __ldg(a.fcn + (size_t)c * hw + p));
    float smax = -INFINITY;
    for (int i = 0; i < a.k; ++i) {
      float seg, msk; bool cov;
      pl_inst_terms(tab[i], a, p, y, x, &seg, &cov, &msk);
      smax = fmaxf(smax, seg);                 // the zeros outside the windows take part (resnet_upsnet.py:163)
      push(a.num_stuff + i, seg + msk);
    }
    if (a.enable_void) {
      float tmax = -INFINITY;
      for (int c = a.num_stuff; c < a.S; ++c) tmax = fmaxf(tmax, __ldg(a.fcn + (size_t)c * hw + p));
      push(a.num_stuff + a.k, tmax - smax);
    }
    const float lse = m + logf(s);
    const bool valid = g >= 0 && g < nch && g != 255;
    a.lse[p] = lse;
    a.gtc[p] = g == 255 ? 255 : (valid ? (int)g : kPlInvalid);
    if (valid) loss[0] = (double)(lse - lg);
    cnt[0] = am == g;
    cnt[1] = g == 255;
  }
  cta_partials<kPlThreads, 1, 2>(loss, cnt, a.part_loss, a.part_cnt);
}

// second stage: one CTA sums the block partials in a fixed order
__global__ void __launch_bounds__(kPlThreads) pl_finish_kernel(const double* part_loss, const int* part_cnt, int nblocks, int hw,
                                                               float* loss, float* accuracy, int* counts) {
  double l[1];
  int c[2];
  cta_sum_partials<kPlThreads, 1, 2>(part_loss, part_cnt, nblocks, l, c);
  if (threadIdx.x == 0) {
    *loss = (float)(l[0] / (double)hw);                                   // .mean() over all pixels, ignored included
    *accuracy = __fdiv_rn((float)c[0], (float)(hw - c[1]));               // correct.float() / total.float()
    counts[0] = c[0];
    counts[1] = c[1];
  }
}

// d fcn_score: the owner of a pixel writes all S channels, zeros included
__global__ void __launch_bounds__(kPlThreads) pl_map_grad_kernel(PlArgs a) {
  extern __shared__ PlInst s_tab[];
  const PlInst* tab = pl_stage_table(a, s_tab);
  const int hw = a.h * a.w, p = blockIdx.x * kPlThreads + threadIdx.x;
  if (p >= hw) return;
  float* d = a.dfcn + p;
  const int g = a.gtc[p];
  if (g == 255 || g == kPlInvalid) {
    for (int c = 0; c < a.S; ++c) d[(size_t)c * hw] = 0.f;
    return;
  }
  const int y = p / a.w, x = p - y * a.w;
  const float lse = a.lse[p], sc = __fdiv_rn(*a.grad_out, (float)hw);
  auto grad = [&](int c, float v) { return __fmul_rn(expf(v - lse) - (c == g ? 1.f : 0.f), sc); };
  for (int c = 0; c < a.num_stuff; ++c) d[(size_t)c * hw] = grad(c, __ldg(a.fcn + (size_t)c * hw + p));
  float tmax = -INFINITY;
  int targ = a.num_stuff;
  for (int c = a.num_stuff; c < a.S; ++c) {
    const float v = __ldg(a.fcn + (size_t)c * hw + p);
    if (v > tmax) { tmax = v; targ = c; }
    d[(size_t)c * hw] = 0.f;
  }
  // thing channels: this thread accumulates into its own pixel, instance by instance
  float smax = -INFINITY;
  int win = -1;
  for (int i = 0; i < a.k; ++i) {
    float seg, msk; bool cov;
    pl_inst_terms(tab[i], a, p, y, x, &seg, &cov, &msk);
    if (seg > smax) { smax = seg; win = cov ? i : -1; }
    if (cov) d[(size_t)tab[i].tch * hw] += grad(a.num_stuff + i, seg + msk);
  }
  if (a.enable_void && a.S > a.num_stuff) {
    const float gv = grad(a.num_stuff + a.k, tmax - smax);
    d[(size_t)targ * hw] += gv;
    if (win >= 0) d[(size_t)tab[win].tch * hw] -= gv;     // nothing when the winner is one of the zeros
  }
}

// destination indices d in [0, n) whose two taps can touch source cell v: i0(d) in {v - 1, v}; i0 is monotone in d, so
// they are one interval.  An estimate from the inverse map, then corrected with the forward rule itself.
__device__ __forceinline__ void pl_range(int v, int n, float scale, int M, int* lo_, int* hi_) {
  int lo = (int)floorf(((float)v - 0.5f) / scale - 0.5f);
  lo = min(max(lo, 0), n);
  while (lo > 0 && pl_i0(lo - 1, scale, M) >= v - 1) --lo;
  while (lo < n && pl_i0(lo, scale, M) < v - 1) ++lo;
  int hi = (int)ceilf(((float)v + 1.5f) / scale - 0.5f);
  hi = min(max(hi, -1), n - 1);
  while (hi < n - 1 && pl_i0(hi + 1, scale, M) <= v) ++hi;
  while (hi >= 0 && pl_i0(hi, scale, M) > v) --hi;
  *lo_ = lo; *hi_ = hi;
}

// d mask_score as a gather: CTA (instance i, source row v), lane u owns source cell (v, u) and sums, over the rectangle
// of destination pixels that touch it, weight * g recomputed from the saved log-sum-exp.  threadIdx.y splits the
// rectangle's rows four ways; the four partials are added in a fixed order.
__global__ void __launch_bounds__(128) pl_mask_grad_kernel(PlArgs a) {
  __shared__ float s_part[4][32];
  const int i = blockIdx.x, v = blockIdx.y, u = threadIdx.x, part = threadIdx.y;
  const PlInst t = a.tab[i];
  const int hw = a.h * a.w, M = a.M, ch = a.num_stuff + i;
  float acc = 0.f;
  if (u < M) {
    int ylo, yhi, xlo, xhi;
    pl_range(v, t.bh, t.scy, M, &ylo, &yhi);
    pl_range(u, t.bw, t.scx, M, &xlo, &xhi);
    ylo = max(ylo, -t.my0); yhi = min(yhi, t.ey - 1 - t.my0);      // crop to the image
    xlo = max(xlo, -t.mx0); xhi = min(xhi, t.ex - 1 - t.mx0);
    for (int dy = ylo + part; dy <= yhi; dy += 4) {
      const int y = t.my0 + dy;
      const PlTap ty = pl_tap(dy, t.scy, M);
      const float wy = (ty.i0 == v ? ty.l0 : 0.f) + (ty.i1 == v ? ty.l1 : 0.f);
      const bool rowcov = y >= t.sy0 && y < t.sy1;
      for (int dx = xlo; dx <= xhi; ++dx) {
        const int x = t.mx0 + dx, p = y * a.w + x;
        const int g = a.gtc[p];
        if (g == 255 || g == kPlInvalid) continue;
        const PlTap tx = pl_tap(dx, t.scx, M);
        const float wx = (tx.i0 == u ? tx.l0 : 0.f) + (tx.i1 == u ? tx.l1 : 0.f);
        const float seg = (rowcov && x >= t.sx0 && x < t.sx1) ? __ldg(a.fcn + (size_t)t.tch * hw + p) : 0.f;
        const float logit = seg + pl_mask_value(a.mask + t.moff, M, ty, tx);
        acc = __fmaf_rn(__fmul_rn(wy, wx), expf(logit - a.lse[p]) - (g == ch ? 1.f : 0.f), acc);
      }
    }
  }
  s_part[part][threadIdx.x] = acc;
  __syncthreads();
  if (part == 0 && u < M) {
    const float sum = ((s_part[0][u] + s_part[1][u]) + s_part[2][u]) + s_part[3][u];
    a.dmask[t.moff + v * M + u] = __fmul_rn(sum, __fdiv_rn(*a.grad_out, (float)hw));
  }
}

template <typename MT>
__global__ void __launch_bounds__(kPlThreads) pl_gt_kernel(const int64_t* seg_gt, const MT* mask_gt, const int64_t* keep, int n,
                                                           int G, int hw, int num_stuff, int64_t* out) {
  const int p = blockIdx.x * kPlThreads + threadIdx.x;
  if (p < hw) out[p] = pl_gt_value<MT>(seg_gt, mask_gt, keep, n, G, hw, p, num_stuff);
}

__global__ void pl_draw_keys_kernel(unsigned long long seed, int stream_id, int n, unsigned long long* keys) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) keys[p] = draw_key(seed, stream_id, (unsigned long long)p);
}

inline int pl_blocks(int h, int w) { return (int)(((size_t)h * w + kPlThreads - 1) / kPlThreads); }

inline size_t pl_layout(int k, int h, int w, void* base, PlArgs& a) {
  const int nblocks = pl_blocks(h, w);
  WsCarve c(base);
  a.tab = c.take<PlInst>(k);
  a.part_loss = c.take<double>(nblocks);
  a.part_cnt = c.take<int>((size_t)nblocks * 2);
  return c.bytes();
}

// argument checks, the workspace carve and the instance table shared by forward and backward
int pl_prepare(PlArgs& a, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  if (!a.fcn || !a.mask || !a.rois || !a.cls || !workspace) return UPSNET_E_BADARG;
  if (a.S <= 0 || a.h <= 0 || a.w <= 0 || a.k <= 0 || a.M <= 0 || a.num_classes <= 0 || a.num_classes > a.S ||
      (a.C != 1 && a.C != a.num_classes) || !(a.box_scale > 0.f))
    return UPSNET_E_BADARG;
  if (a.M > kPlMaxM || (size_t)a.S * a.h * a.w >= (1ull << 31) || (size_t)a.k * a.C * a.M * a.M >= (1ull << 31))
    return UPSNET_E_UNSUPPORTED;
  if (workspace_bytes < pl_layout(a.k, a.h, a.w, workspace, a)) return UPSNET_E_WORKSPACE;
  a.num_stuff = a.S - a.num_classes + 1;
  a.tab_smem = (size_t)a.k * sizeof(PlInst) <= kPlSmemTable;
  pl_table_kernel<<<ceil_div(a.k, 128), 128, 0, st>>>(a);
  UPS_CHECK_LAUNCH();
  return 0;
}

}  // namespace
}  // namespace ups

extern "C" int upsnet_panoptic_loss_workspace_bytes(int k, int h, int w, size_t* bytes) {
  if (!bytes || k <= 0 || h <= 0 || w <= 0) return UPSNET_E_BADARG;
  ups::PlArgs a{};
  *bytes = ups::pl_layout(k, h, w, nullptr, a);
  return 0;
}

extern "C" int upsnet_panoptic_loss_forward(const float* fcn_score, int S, int h, int w, const float* mask_score, int k, int C,
                                            int mask_size, const float* gt_rois, const int64_t* cls_idx,
                                            const int64_t* seg_gt, const void* mask_gt, int mask_gt_is_int64, int G,
                                            const int64_t* keep_inds, int num_classes, int enable_void, float box_scale,
                                            float* loss, float* accuracy, int* counts, float* lse, int* gt_channel,
                                            void* workspace, size_t workspace_bytes, void* stream) {
  using namespace ups;
  if (!seg_gt || !mask_gt || !loss || !accuracy || !counts || !lse || !gt_channel || G <= 0) return UPSNET_E_BADARG;
  if (!keep_inds && G != k) return UPSNET_E_BADARG;      // without a draw, instance channel i is ground-truth mask i
  PlArgs a{};
  a.fcn = fcn_score; a.mask = mask_score; a.rois = gt_rois; a.cls = cls_idx; a.seg_gt = seg_gt; a.mask_gt = mask_gt;
  a.keep = keep_inds;
  a.S = S; a.h = h; a.w = w; a.k = k; a.C = C; a.M = mask_size; a.G = G; a.num_classes = num_classes;
  a.enable_void = enable_void ? 1 : 0; a.box_scale = box_scale;
  a.lse = lse; a.gtc = gt_channel;
  cudaStream_t st = (cudaStream_t)stream;
  const int rc = pl_prepare(a, workspace, workspace_bytes, st);
  if (rc) return rc;
  const int nblocks = pl_blocks(h, w);
  const size_t smem = a.tab_smem ? (size_t)k * sizeof(PlInst) : 0;
  if (mask_gt_is_int64)
    pl_forward_kernel<int64_t><<<nblocks, kPlThreads, smem, st>>>(a);
  else
    pl_forward_kernel<unsigned char><<<nblocks, kPlThreads, smem, st>>>(a);
  UPS_CHECK_LAUNCH();
  pl_finish_kernel<<<1, kPlThreads, 0, st>>>(a.part_loss, a.part_cnt, nblocks, h * w, loss, accuracy, counts);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_panoptic_loss_backward(const float* fcn_score, int S, int h, int w, const float* mask_score, int k, int C,
                                             int mask_size, const float* gt_rois, const int64_t* cls_idx, int num_classes,
                                             int enable_void, float box_scale, const float* lse, const int* gt_channel,
                                             const float* grad_out, float* d_fcn_score, float* d_mask_score,
                                             void* workspace, size_t workspace_bytes, void* stream) {
  using namespace ups;
  if (!lse || !gt_channel || !grad_out || (!d_fcn_score && !d_mask_score)) return UPSNET_E_BADARG;
  PlArgs a{};
  a.fcn = fcn_score; a.mask = mask_score; a.rois = gt_rois; a.cls = cls_idx;
  a.S = S; a.h = h; a.w = w; a.k = k; a.C = C; a.M = mask_size; a.num_classes = num_classes;
  a.enable_void = enable_void ? 1 : 0; a.box_scale = box_scale;
  a.lse = const_cast<float*>(lse); a.gtc = const_cast<int*>(gt_channel);
  a.grad_out = grad_out; a.dfcn = d_fcn_score; a.dmask = d_mask_score;
  cudaStream_t st = (cudaStream_t)stream;
  const int rc = pl_prepare(a, workspace, workspace_bytes, st);
  if (rc) return rc;
  if (d_fcn_score) {
    const size_t smem = a.tab_smem ? (size_t)k * sizeof(PlInst) : 0;
    pl_map_grad_kernel<<<pl_blocks(h, w), kPlThreads, smem, st>>>(a);
    UPS_CHECK_LAUNCH();
  }
  if (d_mask_score) {
    if (C > 1) UPS_CUDA(cudaMemsetAsync(d_mask_score, 0, (size_t)k * C * mask_size * mask_size * sizeof(float), st));
    pl_mask_grad_kernel<<<dim3(k, mask_size), dim3(32, 4), 0, st>>>(a);
    UPS_CHECK_LAUNCH();
  }
  return 0;
}

extern "C" int upsnet_panoptic_gt(const int64_t* seg_gt, const void* mask_gt, int mask_gt_is_int64, int G,
                                  const int64_t* keep_inds, int k, int h, int w, int num_seg_classes, int num_classes,
                                  int64_t* panoptic_gt, void* stream) {
  using namespace ups;
  if (!seg_gt || !mask_gt || !panoptic_gt || G <= 0 || h <= 0 || w <= 0 || num_classes <= 0 || num_classes > num_seg_classes ||
      (keep_inds && k <= 0))
    return UPSNET_E_BADARG;
  if ((size_t)h * w >= (1ull << 31)) return UPSNET_E_UNSUPPORTED;
  const int hw = h * w, n = keep_inds ? k : G, num_stuff = num_seg_classes - num_classes + 1;
  cudaStream_t st = (cudaStream_t)stream;
  if (mask_gt_is_int64)
    pl_gt_kernel<int64_t><<<ceil_div(hw, kPlThreads), kPlThreads, 0, st>>>(seg_gt, (const int64_t*)mask_gt, keep_inds, n, G, hw,
                                                                         num_stuff, panoptic_gt);
  else
    pl_gt_kernel<unsigned char><<<ceil_div(hw, kPlThreads), kPlThreads, 0, st>>>(seg_gt, (const unsigned char*)mask_gt,
                                                                               keep_inds, n, G, hw, num_stuff, panoptic_gt);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_draw_keys(unsigned long long seed, int stream_id, int n, unsigned long long* keys, void* stream) {
  if (!keys || n <= 0 || (stream_id != 0 && stream_id != 1)) return UPSNET_E_BADARG;
  ups::pl_draw_keys_kernel<<<ups::ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(seed, stream_id, n, keys);
  UPS_CHECK_LAUNCH();
  return 0;
}
