// train_loss.cu -- the semantic, RPN and Mask R-CNN losses of the TRAINING forward (models/resnet_upsnet.py:127-142),
// forward and backward.  See include/upsnet_b200.h for the contract of every symbol.
//
// Semantic loss: the cross-entropy (ignore 255) of the x4 bilinear up-sampling of fcn_score, with the up-sampled logits
// evaluated in place through up4.cuh (bit-identical to upsample_bilinear_nchw_kernel) and never stored.  Forward keeps the
// log-sum-exp of every output pixel (4 bytes) for backward; backward is the transpose of the up-sampling applied to the
// per-pixel softmax gradient, computed as a gather over a source tile and its output halo in shared memory.
//
// FCN ROI loss (train.fcn_with_roi_loss, models/fcn.py:102-106 + models/resnet_upsnet.py:132-134): the cross-entropy of
// the score conv applied to RoIAlign(28x28, 1/4) of the 512-channel concat of the semantic head.  The score conv and
// ROIAlign are both linear and act on different axes, so the loss samples the S-plane fcn_score instead (plus the share
// of the score bias that ROIAlign's out-of-map zeros remove); backward is a gather over the ROI samples that reach each
// fcn_score pixel, the taps re-derived with the forward's rule (roi_sample.cuh).
//
// Determinism: every output element has one owner thread that sums in a fixed order; the scalar losses go through
// per-block partials and a fixed-order second stage.  There is no atomic in this file.
#include "common.cuh"
#include "cta.cuh"
#include "roi_sample.cuh"
#include "up4.cuh"

namespace ups {
namespace {

constexpr int kTlThreads = 256;

inline int tl_blocks(long long n) { return (int)((n + kTlThreads - 1) / kTlThreads); }

// ================================================================================================
// semantic loss
// ================================================================================================
constexpr int kSemNone = -1;      // ignored (255), invalid, or outside the image: no loss, no gradient
constexpr int kSemInvalid = -2;   // neither 255 nor a channel: counted in counts[1]

template <typename LT>
__device__ __forceinline__ int sem_target(const LT* seg, size_t o, int S) {
  const long long v = (long long)seg[o];
  if (v == 255) return kSemNone;
  return (v >= 0 && v < S) ? (int)v : kSemInvalid;
}

// one thread per output quad (output row yo, columns 4q..4q+3): a streaming log-sum-exp over the channels of the four
// up-sampled logits, the loss of the pixels with a target, and the lse of all four (0 where nothing reads it)
template <typename LT>
__global__ void __launch_bounds__(kTlThreads) sem_forward_kernel(const float* __restrict__ fcn, int S, int h, int w,
                                                                const LT* __restrict__ seg, float* __restrict__ lse,
                                                                double* part_d, int* part_i) {
  const int i = blockIdx.x * kTlThreads + threadIdx.x;
  double d[1] = {0.0};
  int n[2] = {0, 0};
  if (i < 4 * h * w) {
    const int yo = i / w, q = i - yo * w;
    const size_t o = (size_t)yo * (4 * w) + 4 * q;
    int t[4];
    bool any = false;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      t[j] = sem_target<LT>(seg, o + j, S);
      any |= t[j] >= 0;
      n[0] += t[j] >= 0;
      n[1] += t[j] == kSemInvalid;
    }
    float4 out = make_float4(0.f, 0.f, 0.f, 0.f);
    if (any) {
      const Up4Row r = up4_row(yo, h);
      const size_t hw = (size_t)h * w;
      float m[4], s[4], lt[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) m[j] = -INFINITY, s[j] = 0.f, lt[j] = 0.f;
      for (int c = 0; c < S; ++c) {
        const float* pl = fcn + c * hw;
        float v[4];
        up4_quad(pl + (size_t)r.y0 * w, pl + (size_t)r.y1 * w, q, w, r.ly, r.hy, v);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (v[j] > m[j]) { s[j] = __fmaf_rn(s[j], expf(m[j] - v[j]), 1.f); m[j] = v[j]; }
          else s[j] += expf(v[j] - m[j]);
          if (c == t[j]) lt[j] = v[j];
        }
      }
      float l[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        l[j] = m[j] + logf(s[j]);
        if (t[j] >= 0) d[0] += (double)(l[j] - lt[j]);
      }
      out = make_float4(l[0], l[1], l[2], l[3]);
    }
    *reinterpret_cast<float4*>(lse + o) = out;
  }
  cta_partials<kTlThreads, 1, 2>(d, n, part_d, part_i);
}

__global__ void __launch_bounds__(kTlThreads) sem_finish_kernel(const double* part_d, const int* part_i, int nblocks,
                                                                float* loss, int* counts) {
  double d[1];
  int n[2];
  cta_sum_partials<kTlThreads, 1, 2>(part_d, part_i, nblocks, d, n);
  if (threadIdx.x == 0) {
    *loss = (float)(d[0] / (double)n[0]);          // 0 / 0 = NaN when every pixel is ignored, as torch's mean
    counts[0] = n[0];
    counts[1] = n[1];
  }
}

// backward tile: kSbTy x kSbTx source pixels.  Source row y receives from output rows 4y-2 .. 4y+5, so the tile's output
// halo is rows 4*y0-2 .. 4*(y0+kSbTy)+1 (kSbOr) and the output quads x0-1 .. x0+kSbTx (kSbOc columns, from 4*(x0-1)).
constexpr int kSbTx = 32, kSbTy = 8;
constexpr int kSbOr = 4 * kSbTy + 4;
constexpr int kSbQ = kSbTx + 2;
constexpr int kSbOc = 4 * kSbQ;
constexpr size_t kSbSmem = (size_t)kSbOr * kSbOc * (2 * sizeof(float) + sizeof(short)) + (size_t)kSbOr * kSbTx * sizeof(float);

// d fcn_score[c] = scale * sum over outputs o of w(o -> source) * (softmax_c(o) - [c = t(o)]): per channel, the softmax
// gradient of the halo (one exp per output pixel), then the transpose of the up-sampling, first along x, then along y,
// with the tap weights of up4_row (the same rule as the forward's in both directions).
template <typename LT>
__global__ void __launch_bounds__(kTlThreads) sem_backward_kernel(const float* __restrict__ fcn, int S, int h, int w,
                                                                 const LT* __restrict__ seg, const float* __restrict__ lse,
                                                                 const int* __restrict__ counts,
                                                                 const float* __restrict__ grad_out, float* __restrict__ dfcn) {
  extern __shared__ float4 s_raw[];
  float* s_lse = reinterpret_cast<float*>(s_raw);
  float* s_g = s_lse + kSbOr * kSbOc;
  float* s_xr = s_g + kSbOr * kSbOc;
  short* s_t = reinterpret_cast<short*>(s_xr + kSbOr * kSbTx);
  const int x0 = blockIdx.x * kSbTx, y0 = blockIdx.y * kSbTy, tid = threadIdx.x;
  const int H4 = 4 * h, W4 = 4 * w, oy0 = 4 * y0 - 2, ox0 = 4 * (x0 - 1);
  const size_t hw = (size_t)h * w;
  for (int e = tid; e < kSbOr * kSbOc; e += kTlThreads) {
    const int r = e / kSbOc, j = e - r * kSbOc, oy = oy0 + r, ox = ox0 + j;
    int t = kSemNone;
    float l = 0.f;
    if (oy >= 0 && oy < H4 && ox >= 0 && ox < W4) {
      const size_t o = (size_t)oy * W4 + ox;
      t = max(sem_target<LT>(seg, o, S), kSemNone);
      if (t >= 0) l = lse[o];
    }
    s_t[e] = (short)t;
    s_lse[e] = l;
  }
  __syncthreads();
  const int N = counts[0];
  const float scale = N > 0 ? __fdiv_rn(*grad_out, (float)N) : 0.f;
  const int sx = tid & (kSbTx - 1), sy = tid / kSbTx;
  const int x = x0 + sx, y = y0 + sy;
  for (int c = 0; c < S; ++c) {
    const float* pl = fcn + c * hw;
    // A: softmax gradient of channel c over the halo, one quad per item
    for (int e = tid; e < kSbOr * kSbQ; e += kTlThreads) {
      const int r = e / kSbQ, jq = e - r * kSbQ, q = x0 - 1 + jq, oy = oy0 + r;
      float* g = s_g + r * kSbOc + 4 * jq;
      const short* t = s_t + r * kSbOc + 4 * jq;
      const float* l = s_lse + r * kSbOc + 4 * jq;
      if (t[0] < 0 && t[1] < 0 && t[2] < 0 && t[3] < 0) {     // also every quad outside the image
        g[0] = g[1] = g[2] = g[3] = 0.f;
        continue;
      }
      const Up4Row rw = up4_row(oy, h);
      float v[4];
      up4_quad(pl + (size_t)rw.y0 * w, pl + (size_t)rw.y1 * w, q, w, rw.ly, rw.hy, v);
#pragma unroll
      for (int j = 0; j < 4; ++j) g[j] = t[j] >= 0 ? expf(v[j] - l[j]) - (c == t[j] ? 1.f : 0.f) : 0.f;
    }
    __syncthreads();
    // B: along x, source column x0 + bx receives from output columns 4x-2 .. 4x+5 (halo columns 4bx+2 .. 4bx+9)
    for (int e = tid; e < kSbOr * kSbTx; e += kTlThreads) {
      const int r = e / kSbTx, bx = e - r * kSbTx, xs = x0 + bx;
      float acc = 0.f;
      if (xs < w) {
        const float* g = s_g + r * kSbOc;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int ox = 4 * xs - 2 + k;
          if (ox < 0 || ox >= W4) continue;
          const Up4Row tp = up4_row(ox, w);
          const float wt = (tp.y0 == xs ? tp.hy : 0.f) + (tp.y1 == xs ? tp.ly : 0.f);
          acc = __fmaf_rn(wt, g[4 * bx + 2 + k], acc);
        }
      }
      s_xr[e] = acc;
    }
    __syncthreads();
    // C: along y, one source pixel per thread
    if (x < w && y < h) {
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int oy = 4 * y - 2 + k;
        if (oy < 0 || oy >= H4) continue;
        const Up4Row tp = up4_row(oy, h);
        const float wt = (tp.y0 == y ? tp.hy : 0.f) + (tp.y1 == y ? tp.ly : 0.f);
        acc = __fmaf_rn(wt, s_xr[(4 * sy + k) * kSbTx + sx], acc);
      }
      dfcn[c * hw + (size_t)y * w + x] = __fmul_rn(acc, scale);
    }
    // the next channel's phase A writes s_g only: every thread has passed the barrier after phase B
  }
}

inline size_t sem_layout(int h, int w, void* base, double** pd, int** pi) {
  const int nblocks = tl_blocks(4ll * h * w);
  WsCarve c(base);
  *pd = c.take<double>(nblocks);
  *pi = c.take<int>((size_t)nblocks * 2);
  return c.bytes();
}

int sem_check(const float* fcn, int S, int h, int w, const void* seg) {
  if (!fcn || !seg || S <= 0 || h <= 0 || w <= 0) return UPSNET_E_BADARG;
  if ((size_t)S * h * w >= (1ull << 31) || 16ull * h * w >= (1ull << 31) || S > 32767) return UPSNET_E_UNSUPPORTED;
  return 0;
}

// ================================================================================================
// RPN loss
// ================================================================================================
constexpr int kRpnMaxLevels = 8;

struct RpnLevel {
  const float* score; const float* pred; const int64_t* label; const float* tgt; const float* iw; const float* ow;
  float* dscore; float* dpred;
  long long lsc, lsy, bsc, bsy;   // channel / row strides (elements) of the label field and of the three box fields
  int h, w, begin;                // score map size; first anchor index of the level
};

struct RpnArgs {
  RpnLevel lv[kRpnMaxLevels];
  int L, A, total;
  float batch;
};

// the level, channel and pixel of anchor index i
__device__ __forceinline__ const RpnLevel& rpn_locate(const RpnArgs& a, int i, int* an, int* y, int* x) {
  int l = 0;
  for (int k = 1; k < a.L; ++k) l = i >= a.lv[k].begin ? k : l;
  const RpnLevel& v = a.lv[l];
  const int hw = v.h * v.w, loc = i - v.begin;
  *an = loc / hw;
  const int pix = loc - *an * hw;
  *y = pix / v.w;
  *x = pix - *y * v.w;
  return v;
}

// F.binary_cross_entropy_with_logits, ATen's formula: (1 - t) x + m + log(exp(-m) + exp(-x - m)), m = max(-x, 0)
__device__ __forceinline__ float rpn_bce(float x, float t) {
  const float m = fmaxf(-x, 0.f);
  return (1.f - t) * x + m + logf(expf(-m) + expf(-x - m));
}

__global__ void __launch_bounds__(kTlThreads) rpn_forward_kernel(RpnArgs a, double* part_d, int* part_i) {
  const int i = blockIdx.x * kTlThreads + threadIdx.x;
  double d[2] = {0.0, 0.0};
  int n[1] = {0};
  if (i < a.total) {
    int an, y, x;
    const RpnLevel& v = rpn_locate(a, i, &an, &y, &x);
    const size_t hw = (size_t)v.h * v.w, pix = (size_t)y * v.w + x;
    const long long lab = v.label[an * v.lsc + y * v.lsy + x];
    if (lab != -1) {
      d[0] = (double)rpn_bce(__ldg(v.score + an * hw + pix), (float)lab);
      n[0] = 1;
    }
    float bl = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int ch = 4 * an + k;
      const long long f = ch * v.bsc + y * v.bsy + x;
      const float iw = __ldg(v.iw + f), ow = __ldg(v.ow + f);
      const float dd = iw * (__ldg(v.pred + ch * hw + pix) - __ldg(v.tgt + f)), ad = fabsf(dd);
      // sigma 3: 0.5 sigma^2 d^2 inside |d| < 1 / sigma^2, |d| - 0.5 / sigma^2 outside
      bl += (ad < 1.f / 9.f ? dd * dd * 4.5f : ad - 0.5f / 9.f) * ow;
    }
    d[1] = (double)bl;
  }
  cta_partials<kTlThreads, 2, 1>(d, n, part_d, part_i);
}

__global__ void __launch_bounds__(kTlThreads) rpn_finish_kernel(const double* part_d, const int* part_i, int nblocks,
                                                                float batch, float* cls_loss, float* bbox_loss) {
  double d[2];
  int n[1];
  cta_sum_partials<kTlThreads, 2, 1>(part_d, part_i, nblocks, d, n);
  if (threadIdx.x == 0) {
    *cls_loss = (float)(d[0] / (double)batch);
    *bbox_loss = (float)d[1];
  }
}

__global__ void __launch_bounds__(kTlThreads) rpn_backward_kernel(RpnArgs a, const float* __restrict__ grad_cls,
                                                                 const float* __restrict__ grad_bbox) {
  const int i = blockIdx.x * kTlThreads + threadIdx.x;
  if (i >= a.total) return;
  int an, y, x;
  const RpnLevel& v = rpn_locate(a, i, &an, &y, &x);
  const size_t hw = (size_t)v.h * v.w, pix = (size_t)y * v.w + x;
  if (v.dscore) {
    const long long lab = v.label[an * v.lsc + y * v.lsy + x];
    float g = 0.f;
    if (lab != -1) {
      const float s = 1.f / (1.f + expf(-__ldg(v.score + an * hw + pix)));
      g = __fmul_rn(s - (float)lab, __fdiv_rn(*grad_cls, a.batch));
    }
    v.dscore[an * hw + pix] = g;
  }
  if (v.dpred) {
    const float gb = *grad_bbox;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int ch = 4 * an + k;
      const long long f = ch * v.bsc + y * v.bsy + x;
      const float iw = __ldg(v.iw + f), ow = __ldg(v.ow + f);
      const float dd = iw * (__ldg(v.pred + ch * hw + pix) - __ldg(v.tgt + f));
      const float dl = fabsf(dd) < 1.f / 9.f ? 9.f * dd : (dd > 0.f ? 1.f : (dd < 0.f ? -1.f : 0.f));
      v.dpred[ch * hw + pix] = dl * ow * iw * gb;
    }
  }
}

inline size_t rpn_layout(int total, void* base, double** pd, int** pi) {
  const int nblocks = tl_blocks(total);
  WsCarve c(base);
  *pd = c.take<double>((size_t)nblocks * 2);
  *pi = c.take<int>(nblocks);
  return c.bytes();
}

int rpn_args(RpnArgs& a, int L, int A, const int* h, const int* w, const float* const* score, const float* const* pred,
             const int64_t* const* labels, const long long* label_strides, const float* const* tgt,
             const float* const* iw, const float* const* ow, const long long* bbox_strides, float batch) {
  if (L <= 0 || A <= 0 || !h || !w || !score || !pred || !labels || !label_strides || !tgt || !iw || !ow ||
      !bbox_strides || !(batch > 0.f))
    return UPSNET_E_BADARG;
  if (L > kRpnMaxLevels) return UPSNET_E_UNSUPPORTED;
  a.L = L; a.A = A; a.batch = batch;
  long long total = 0;
  for (int l = 0; l < L; ++l) {
    RpnLevel& v = a.lv[l];
    v.score = score[l]; v.pred = pred[l]; v.label = labels[l]; v.tgt = tgt[l]; v.iw = iw[l]; v.ow = ow[l];
    v.h = h[l]; v.w = w[l];
    v.lsc = label_strides[2 * l]; v.lsy = label_strides[2 * l + 1];
    v.bsc = bbox_strides[2 * l]; v.bsy = bbox_strides[2 * l + 1];
    if (!v.score || !v.pred || !v.label || !v.tgt || !v.iw || !v.ow || v.h <= 0 || v.w <= 0) return UPSNET_E_BADARG;
    // a field at least as large as the map: rows of >= w elements, channels of >= h rows
    if (v.lsy < v.w || v.lsc < (long long)v.h * v.lsy || v.bsy < v.w || v.bsc < (long long)v.h * v.bsy) return UPSNET_E_BADARG;
    if ((long long)4 * A * v.bsc >= (1ll << 40) || (long long)4 * A * v.h * v.w >= (1ll << 31)) return UPSNET_E_UNSUPPORTED;
    v.begin = (int)total;
    total += (long long)A * v.h * v.w;
  }
  if (total >= (1ll << 31)) return UPSNET_E_UNSUPPORTED;
  a.total = (int)total;
  return 0;
}

// ================================================================================================
// Mask R-CNN loss
// ================================================================================================
constexpr int kMrRowsPerBlock = kTlThreads / 32;   // one warp per cls_score row
constexpr int kMrChunk = 8 * kTlThreads;           // elements per block of the bbox and mask parts

struct MrArgs {
  const float* cls; const int64_t* label; const float* pred; const float* tgt; const float* iw; const float* ow;
  const float* mask; const float* mtgt;
  float* dcls; float* dpred; float* dmask;
  long long mask_n;
  int R, K, B, nb_mask, nb_bbox, nb_cls;
};

// row r of cls_score: max, its first index and log-sum-exp over the K classes, in every lane of the warp
__device__ __forceinline__ void mr_row(const MrArgs& a, int r, float* m_, int* am_, float* lse_) {
  const int lane = threadIdx.x & 31;
  const float* x = a.cls + (size_t)r * a.K;
  float m = -INFINITY;
  int am = a.K;
  for (int c = lane; c < a.K; c += 32) {
    const float v = __ldg(x + c);
    if (v > m) { m = v; am = c; }
  }
  for (int o = 16; o; o >>= 1) {
    const float mo = __shfl_xor_sync(0xffffffffu, m, o);
    const int ao = __shfl_xor_sync(0xffffffffu, am, o);
    if (mo > m || (mo == m && ao < am)) { m = mo; am = ao; }
  }
  float s = 0.f;
  for (int c = lane; c < a.K; c += 32) s += expf(__ldg(x + c) - m);
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  *m_ = m; *am_ = am; *lse_ = m + logf(s);
}

__device__ __forceinline__ float mr_smooth_l1(float p, float t, float iw, float ow) {
  const float d = iw * (p - t), ad = fabsf(d);
  return (ad < 1.f ? d * d * 0.5f : ad - 0.5f) * ow;                  // sigma 1
}

// mask_loss term: -x (t - b) + log(1 + exp(x - 2 x b)), b = (x >= 0); the exponent is -|x|
__device__ __forceinline__ float mr_mask_term(float x, float t) {
  const float b = x >= 0.f ? 1.f : 0.f;
  return -x * (t - b) + log1pf(expf(-fabsf(x)));
}

// blocks [0, nb_mask) the mask elements, then nb_bbox blocks of box elements, then nb_cls blocks of cls rows.
// partials: d = (cls loss, bbox loss, mask loss), n = (rows with a target, rows labelled -1, rows whose arg-max equals the
// label, mask elements with a target)
__global__ void __launch_bounds__(kTlThreads) mr_forward_kernel(MrArgs a, double* part_d, int* part_i) {
  double d[3] = {0.0, 0.0, 0.0};
  int n[4] = {0, 0, 0, 0};
  int b = blockIdx.x;
  if (b < a.nb_mask) {
    float acc = 0.f;
    const long long base = (long long)b * kMrChunk + threadIdx.x;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const long long e = base + k * kTlThreads;
      if (e >= a.mask_n) break;
      const float t = __ldg(a.mtgt + e);
      if (t != -1.f) { acc += mr_mask_term(__ldg(a.mask + e), t); ++n[3]; }
    }
    d[2] = acc;
  } else if ((b -= a.nb_mask) < a.nb_bbox) {
    float acc = 0.f;
    const long long base = (long long)b * kMrChunk + threadIdx.x, total = (long long)a.R * a.B;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const long long e = base + k * kTlThreads;
      if (e >= total) break;
      acc += mr_smooth_l1(__ldg(a.pred + e), __ldg(a.tgt + e), __ldg(a.iw + e), __ldg(a.ow + e));
    }
    d[1] = acc;
  } else {
    b -= a.nb_bbox;
    const int r = b * kMrRowsPerBlock + (threadIdx.x >> 5);
    if (r < a.R) {
      float m, lse;
      int am;
      mr_row(a, r, &m, &am, &lse);
      const long long lab = a.label[r];
      if ((threadIdx.x & 31) == 0) {
        if (lab == -1) n[1] = 1;
        else if (lab >= 0 && lab < a.K) { n[0] = 1; d[0] = (double)(lse - __ldg(a.cls + (size_t)r * a.K + lab)); }
        n[2] = am == lab;
      }
    }
  }
  cta_partials<kTlThreads, 3, 4>(d, n, part_d, part_i);
}

__global__ void __launch_bounds__(kTlThreads) mr_finish_kernel(const double* part_d, const int* part_i, int nblocks, int R,
                                                               float* cls_loss, float* bbox_loss, float* mask_loss,
                                                               float* accuracy, int* counts) {
  double d[3];
  int n[4];
  cta_sum_partials<kTlThreads, 3, 4>(part_d, part_i, nblocks, d, n);
  if (threadIdx.x == 0) {
    *cls_loss = (float)(d[0] / (double)n[0]);                               // mean over rows with a target
    *bbox_loss = (float)(d[1] / (double)R);                                 // loss_box.sum() / loss_box.shape[0]
    *mask_loss = __fdiv_rn((float)d[2], __fadd_rn((float)n[3], 1e-10f));    // / (mask_weight.sum() + 1e-10), float32
    *accuracy = __fdiv_rn((float)(n[2] - n[1]), (float)(R - n[1]));        // rcnn_accuracy, as written
    for (int j = 0; j < 4; ++j) counts[j] = n[j];
  }
}

__global__ void __launch_bounds__(kTlThreads) mr_backward_kernel(MrArgs a, const int* __restrict__ counts,
                                                                const float* __restrict__ grad_cls,
                                                                const float* __restrict__ grad_bbox,
                                                                const float* __restrict__ grad_mask) {
  int b = blockIdx.x;
  if (b < a.nb_mask) {
    if (!a.dmask) return;
    const float s = __fdiv_rn(*grad_mask, __fadd_rn((float)counts[3], 1e-10f));
    const long long base = (long long)b * kMrChunk + threadIdx.x;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const long long e = base + k * kTlThreads;
      if (e >= a.mask_n) break;
      const float t = __ldg(a.mtgt + e);
      float g = 0.f;
      if (t != -1.f) g = __fmul_rn(1.f / (1.f + expf(-__ldg(a.mask + e))) - t, s);
      a.dmask[e] = g;
    }
  } else if ((b -= a.nb_mask) < a.nb_bbox) {
    if (!a.dpred) return;
    const float s = __fdiv_rn(*grad_bbox, (float)a.R);
    const long long base = (long long)b * kMrChunk + threadIdx.x, total = (long long)a.R * a.B;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const long long e = base + k * kTlThreads;
      if (e >= total) break;
      const float iw = __ldg(a.iw + e), ow = __ldg(a.ow + e);
      const float dd = iw * (__ldg(a.pred + e) - __ldg(a.tgt + e));
      const float dl = fabsf(dd) < 1.f ? dd : (dd > 0.f ? 1.f : (dd < 0.f ? -1.f : 0.f));
      a.dpred[e] = dl * ow * iw * s;
    }
  } else {
    if (!a.dcls) return;
    b -= a.nb_bbox;
    const int r = b * kMrRowsPerBlock + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (r >= a.R) return;
    const long long lab = a.label[r];
    float* dx = a.dcls + (size_t)r * a.K;
    if (lab < 0 || lab >= a.K) {
      for (int c = lane; c < a.K; c += 32) dx[c] = 0.f;
      return;
    }
    float m, lse;
    int am;
    mr_row(a, r, &m, &am, &lse);
    const float s = __fdiv_rn(*grad_cls, (float)counts[0]);      // counts[0] >= 1: this row has a target
    const float* x = a.cls + (size_t)r * a.K;
    for (int c = lane; c < a.K; c += 32) dx[c] = __fmul_rn(expf(__ldg(x + c) - lse) - (c == lab ? 1.f : 0.f), s);
  }
}

inline void mr_grid(MrArgs& a) {
  a.nb_mask = (int)((a.mask_n + kMrChunk - 1) / kMrChunk);
  a.nb_bbox = (int)(((long long)a.R * a.B + kMrChunk - 1) / kMrChunk);
  a.nb_cls = ceil_div(a.R, kMrRowsPerBlock);
}

inline size_t mr_layout(MrArgs& a, void* base, double** pd, int** pi) {
  mr_grid(a);
  const int nblocks = a.nb_mask + a.nb_bbox + a.nb_cls;
  WsCarve c(base);
  *pd = c.take<double>((size_t)nblocks * 3);
  *pi = c.take<int>((size_t)nblocks * 4);
  return c.bytes();
}

int mr_args(MrArgs& a, const float* cls_score, const int64_t* cls_label, int R, int K, const float* bbox_pred,
            const float* bbox_target, const float* iw, const float* ow, int B, const float* mask_score,
            const float* mask_target, long long mask_numel) {
  if (!cls_score || !cls_label || !bbox_pred || !bbox_target || !iw || !ow || R <= 0 || K <= 0 || B <= 0 || mask_numel < 0 ||
      (mask_numel > 0 && (!mask_score || !mask_target)))
    return UPSNET_E_BADARG;
  if ((long long)R * K >= (1ll << 31) || (long long)R * B >= (1ll << 31) || mask_numel >= (1ll << 31))
    return UPSNET_E_UNSUPPORTED;
  a.cls = cls_score; a.label = cls_label; a.pred = bbox_pred; a.tgt = bbox_target; a.iw = iw; a.ow = ow;
  a.mask = mask_score; a.mtgt = mask_target; a.mask_n = mask_numel; a.R = R; a.K = K; a.B = B;
  mr_grid(a);
  return 0;
}


// ================================================================================================
// FCN ROI loss
// ================================================================================================
constexpr int kFrSr = 2;            // sampling ratio: the four samples of a cell stay in registers
constexpr int kFrSamples = kFrSr * kFrSr;
constexpr int kFrMaxR = 1024;       // rois; their bin geometry fits the gather's shared memory
constexpr int kFrMaxM = 64;
constexpr int kFrCh = 8;            // channels per thread of the backward gather

struct FrCell {
  SamplePos s[kFrSamples];
  float corr;                       // 1 - n_inside / count: the share of the score bias that sampling fcn_score misses
};

__device__ __forceinline__ RoiBins fr_bins(const float* rois, int r, int M, float sc) {
  const float* q = rois + (size_t)r * 5;
  return roi_bins(__ldg(q + 1), __ldg(q + 2), __ldg(q + 3), __ldg(q + 4), sc, M, M);
}

// the samples of cell (ph, pw) of a roi, by roi_align_nchw_kernel's rule
__device__ __forceinline__ FrCell fr_cell(const RoiBins& g, int ph, int pw, int h, int w) {
  FrCell c;
  int inside = 0;
#pragma unroll
  for (int iy = 0; iy < kFrSr; ++iy) {
    const float y = roi_sample_coord(g.rsh, ph, g.bsh, iy, kFrSr);
#pragma unroll
    for (int ix = 0; ix < kFrSr; ++ix) {
      const float x = roi_sample_coord(g.rsw, pw, g.bsw, ix, kFrSr);
      c.s[iy * kFrSr + ix] = roi_sample(h, w, y, x);
      inside += roi_sample_inside(h, w, y, x);
    }
  }
  c.corr = 1.f - (float)inside / (float)kFrSamples;
  return c;
}

// the reference's roi score of one channel: RoIAlign of the plane pl, plus bias * corr (exactly 0 inside the map)
__device__ __forceinline__ float fr_value(const FrCell& c, const float* __restrict__ pl, float bias) {
  float acc = 0.f;
#pragma unroll
  for (int q = 0; q < kFrSamples; ++q) {
    const SamplePos& s = c.s[q];
    acc += (s.w00 * __ldg(pl + s.o00) + s.w01 * __ldg(pl + s.o01) + s.w10 * __ldg(pl + s.o10) + s.w11 * __ldg(pl + s.o11));
  }
  return acc / (float)kFrSamples + bias * c.corr;
}

// one thread per roi cell: streaming log-sum-exp over the S roi scores, the loss of a cell with a target
template <typename LT>
__global__ void __launch_bounds__(kTlThreads) fr_forward_kernel(const float* __restrict__ fcn, const float* __restrict__ bias,
                                                               int S, int h, int w, const float* __restrict__ rois, int R,
                                                               int M, float sc, const LT* __restrict__ gt,
                                                               float* __restrict__ lse, double* part_d, int* part_i) {
  const int i = blockIdx.x * kTlThreads + threadIdx.x, mm = M * M;
  double d[1] = {0.0};
  int n[2] = {0, 0};
  if (i < R * mm) {
    const int t = sem_target<LT>(gt, i, S);
    n[0] = t >= 0;
    n[1] = t == kSemInvalid;
    float l = 0.f;
    if (t >= 0) {
      const int r = i / mm, p = i - r * mm, ph = p / M, pw = p - ph * M;
      const FrCell c = fr_cell(fr_bins(rois, r, M, sc), ph, pw, h, w);
      const size_t hw = (size_t)h * w;
      float m = -INFINITY, s = 0.f, lt = 0.f;
      for (int ch = 0; ch < S; ++ch) {
        const float v = fr_value(c, fcn + ch * hw, __ldg(bias + ch));
        if (v > m) { s = __fmaf_rn(s, expf(m - v), 1.f); m = v; }
        else s += expf(v - m);
        if (ch == t) lt = v;
      }
      l = m + logf(s);
      d[0] = (double)(l - lt);
    }
    lse[i] = l;
  }
  cta_partials<kTlThreads, 1, 2>(d, n, part_d, part_i);
}

__global__ void __launch_bounds__(kTlThreads) fr_finish_kernel(const double* part_d, const int* part_i, int nblocks, int cells,
                                                               float* loss, int* counts) {
  double d[1];
  int n[2];
  cta_sum_partials<kTlThreads, 1, 2>(part_d, part_i, nblocks, d, n);
  if (threadIdx.x == 0) {
    *loss = (float)(d[0] / (double)cells);      // reduce=False + .mean(): ignored cells count in the denominator
    counts[0] = n[0];
    counts[1] = n[1];
  }
}

// backward, pass 1: gc[ch][cell] = (softmax_ch - [ch = t]) * grad_out / cells, channel-major; corr[cell] for d bias
template <typename LT>
__global__ void __launch_bounds__(kTlThreads) fr_grad_kernel(const float* __restrict__ fcn, const float* __restrict__ bias,
                                                            int S, int h, int w, const float* __restrict__ rois, int R, int M,
                                                            float sc, const LT* __restrict__ gt, const float* __restrict__ lse,
                                                            const float* __restrict__ grad_out, float* __restrict__ gc,
                                                            float* __restrict__ corr) {
  const int i = blockIdx.x * kTlThreads + threadIdx.x, mm = M * M, cells = R * mm;
  if (i >= cells) return;
  const int t = sem_target<LT>(gt, i, S);
  if (t < 0) {
    for (int ch = 0; ch < S; ++ch) gc[(size_t)ch * cells + i] = 0.f;
    corr[i] = 0.f;
    return;
  }
  const int r = i / mm, p = i - r * mm, ph = p / M, pw = p - ph * M;
  const FrCell c = fr_cell(fr_bins(rois, r, M, sc), ph, pw, h, w);
  const size_t hw = (size_t)h * w;
  const float l = lse[i], scale = __fdiv_rn(*grad_out, (float)cells);
  for (int ch = 0; ch < S; ++ch) {
    const float v = fr_value(c, fcn + ch * hw, __ldg(bias + ch));
    gc[(size_t)ch * cells + i] = __fmul_rn(expf(v - l) - (ch == t ? 1.f : 0.f), scale);
  }
  corr[i] = c.corr;
}

// a candidate sample index, kept in [-2, K] before the conversion to int (far rois give huge quotients)
__device__ __forceinline__ float fr_clampk(float k, int K) { return fminf(fmaxf(k, -2.f), (float)K); }

// backward, pass 2: d fcn_score[c][y][x] = sum over rois in order, then over the samples whose taps can reach (y, x), of
// tap weight * gc[c][cell] / count.  A sample reaches row y only if max(sample y, 0) lies in [y-1, y+1) (below 0 it is
// clamped to 0; at or above h-1 it reads row h-1 alone), so each roi contributes a short range of sample rows and
// columns; every candidate's taps are re-derived with roi_sample, so the weights are the forward's, bit for bit.
__global__ void __launch_bounds__(kTlThreads) fr_gather_kernel(const float* __restrict__ gc, const float* __restrict__ rois,
                                                              int R, int M, float sc, int S, int h, int w,
                                                              float* __restrict__ dfcn) {
  __shared__ float4 s_geo[kFrMaxR];
  __shared__ float2 s_inv[kFrMaxR];     // 1 / sample step along x and y: the candidate ranges need no division
  for (int r = threadIdx.x; r < R; r += kTlThreads) {
    const RoiBins g = fr_bins(rois, r, M, sc);
    s_geo[r] = make_float4(g.rsw, g.rsh, g.bsw, g.bsh);
    s_inv[r] = make_float2(kFrSr / g.bsw, kFrSr / g.bsh);
  }
  __syncthreads();
  const int pix = blockIdx.x * kTlThreads + threadIdx.x;
  if (pix >= h * w) return;
  const int y = pix / w, x = pix - y * w, c0 = blockIdx.y * kFrCh, K = M * kFrSr, cells = R * M * M;
  const float ylo = y <= 1 ? -1.f : (float)(y - 1), yhi = y == h - 1 ? (float)h : (float)(y + 1);
  const float xlo = x <= 1 ? -1.f : (float)(x - 1), xhi = x == w - 1 ? (float)w : (float)(x + 1);
  float acc[kFrCh];
#pragma unroll
  for (int j = 0; j < kFrCh; ++j) acc[j] = 0.f;
  for (int r = 0; r < R; ++r) {
    const float4 g = s_geo[r];
    const float2 inv = s_inv[r];
    // candidate sample indices k = p * kFrSr + i, coordinate ~ start + (k + 0.5) * bin / kFrSr, widened by one (which
    // also covers the rounding of the reciprocal)
    const int ky0 = max((int)floorf(fr_clampk((ylo - g.y) * inv.y - 0.5f, K)) - 1, 0);
    const int ky1 = min((int)ceilf(fr_clampk((yhi - g.y) * inv.y - 0.5f, K)) + 1, K - 1);
    const int kx0 = max((int)floorf(fr_clampk((xlo - g.x) * inv.x - 0.5f, K)) - 1, 0);
    const int kx1 = min((int)ceilf(fr_clampk((xhi - g.x) * inv.x - 0.5f, K)) + 1, K - 1);
    for (int ky = ky0; ky <= ky1; ++ky) {
      const int ph = ky / kFrSr, iy = ky - ph * kFrSr;
      const float ys = roi_sample_coord(g.y, ph, g.w, iy, kFrSr);
      for (int kx = kx0; kx <= kx1; ++kx) {
        const int pw = kx / kFrSr, ix = kx - pw * kFrSr;
        const SamplePos s = roi_sample(h, w, ys, roi_sample_coord(g.x, pw, g.z, ix, kFrSr));
        const float wt = (s.o00 == pix ? s.w00 : 0.f) + (s.o01 == pix ? s.w01 : 0.f) + (s.o10 == pix ? s.w10 : 0.f) +
                         (s.o11 == pix ? s.w11 : 0.f);
        if (wt == 0.f) continue;
        const float* gp = gc + (size_t)c0 * cells + ((size_t)r * M + ph) * M + pw;
#pragma unroll
        for (int j = 0; j < kFrCh; ++j)
          if (c0 + j < S) acc[j] = __fmaf_rn(wt, __ldg(gp + (size_t)j * cells), acc[j]);
      }
    }
  }
  const size_t hw = (size_t)h * w;
#pragma unroll
  for (int j = 0; j < kFrCh; ++j)
    if (c0 + j < S) dfcn[(c0 + j) * hw + pix] = acc[j] * (1.f / kFrSamples);   // count is a power of two: exact
}

// backward, pass 3: d bias[c] = sum over cells of gc[c][cell] * corr[cell] (a fixed-order tree per channel)
__global__ void __launch_bounds__(kTlThreads) fr_dbias_kernel(const float* __restrict__ gc, const float* __restrict__ corr,
                                                             int cells, float* __restrict__ dbias) {
  __shared__ float s_a[kTlThreads];
  const int c = blockIdx.x;
  float a = 0.f;
  for (int i = threadIdx.x; i < cells; i += kTlThreads) {
    const float k = __ldg(corr + i);
    if (k != 0.f) a = __fmaf_rn(__ldg(gc + (size_t)c * cells + i), k, a);
  }
  s_a[threadIdx.x] = a;
  __syncthreads();
  for (int o = kTlThreads / 2; o; o >>= 1) {
    if (threadIdx.x < o) s_a[threadIdx.x] += s_a[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) dbias[c] = s_a[0];
}

inline size_t fr_layout(int S, int R, int M, int backward, void* base, double** pd, int** pi, float** gc, float** corr) {
  const long long cells = (long long)R * M * M;
  WsCarve c(base);
  if (backward) {
    *gc = c.take<float>((size_t)S * cells);
    *corr = c.take<float>((size_t)cells);
  } else {
    const int nblocks = tl_blocks(cells);
    *pd = c.take<double>(nblocks);
    *pi = c.take<int>((size_t)nblocks * 2);
  }
  return c.bytes();
}

int fr_check(const float* fcn, const float* bias, int S, int h, int w, const float* rois, int R, const void* gt, int M,
             int sampling_ratio, float spatial_scale) {
  if (!fcn || !bias || !rois || !gt || S <= 0 || h <= 0 || w <= 0 || R < 0 || M <= 0 || !(spatial_scale > 0.f))
    return UPSNET_E_BADARG;
  if (R == 0 || R > kFrMaxR || M > kFrMaxM || sampling_ratio != kFrSr || (size_t)S * h * w >= (1ull << 31) ||
      (size_t)S * R * M * M >= (1ull << 31) || S > 32767)
    return UPSNET_E_UNSUPPORTED;
  return 0;
}

}  // namespace
}  // namespace ups

// ---- semantic loss -------------------------------------------------------------------------------
extern "C" int upsnet_semantic_loss_workspace_bytes(int h, int w, size_t* bytes) {
  if (!bytes || h <= 0 || w <= 0) return UPSNET_E_BADARG;
  double* pd; int* pi;
  *bytes = ups::sem_layout(h, w, nullptr, &pd, &pi);
  return 0;
}

extern "C" int upsnet_semantic_loss_forward(const float* fcn_score, int S, int h, int w, const void* seg_gt,
                                            int seg_gt_is_int64, float* loss, int* counts, float* lse, void* workspace,
                                            size_t workspace_bytes, void* stream) {
  using namespace ups;
  int rc = sem_check(fcn_score, S, h, w, seg_gt);
  if (rc) return rc;
  if (!loss || !counts || !lse || !workspace || ((uintptr_t)lse & 15)) return UPSNET_E_BADARG;
  double* pd; int* pi;
  if (workspace_bytes < sem_layout(h, w, workspace, &pd, &pi)) return UPSNET_E_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const int nblocks = tl_blocks(4ll * h * w);
  if (seg_gt_is_int64)
    sem_forward_kernel<int64_t><<<nblocks, kTlThreads, 0, st>>>(fcn_score, S, h, w, (const int64_t*)seg_gt, lse, pd, pi);
  else
    sem_forward_kernel<unsigned char><<<nblocks, kTlThreads, 0, st>>>(fcn_score, S, h, w, (const unsigned char*)seg_gt, lse,
                                                                       pd, pi);
  UPS_CHECK_LAUNCH();
  sem_finish_kernel<<<1, kTlThreads, 0, st>>>(pd, pi, nblocks, loss, counts);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_semantic_loss_backward(const float* fcn_score, int S, int h, int w, const void* seg_gt,
                                             int seg_gt_is_int64, const float* lse, const int* counts,
                                             const float* grad_out, float* d_fcn_score, void* stream) {
  using namespace ups;
  int rc = sem_check(fcn_score, S, h, w, seg_gt);
  if (rc) return rc;
  if (!lse || !counts || !grad_out || !d_fcn_score) return UPSNET_E_BADARG;
  static PerDeviceOnce configured;
  if (configured.need()) {
    UPS_CUDA(cudaFuncSetAttribute(sem_backward_kernel<int64_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSbSmem));
    UPS_CUDA(cudaFuncSetAttribute(sem_backward_kernel<unsigned char>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)kSbSmem));
  }
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid(ceil_div(w, kSbTx), ceil_div(h, kSbTy));
  if (seg_gt_is_int64)
    sem_backward_kernel<int64_t><<<grid, kTlThreads, kSbSmem, st>>>(fcn_score, S, h, w, (const int64_t*)seg_gt, lse, counts,
                                                                    grad_out, d_fcn_score);
  else
    sem_backward_kernel<unsigned char><<<grid, kTlThreads, kSbSmem, st>>>(fcn_score, S, h, w, (const unsigned char*)seg_gt,
                                                                          lse, counts, grad_out, d_fcn_score);
  UPS_CHECK_LAUNCH();
  return 0;
}

// ---- RPN loss -----------------------------------------------------------------------------------
extern "C" int upsnet_rpn_loss_workspace_bytes(int num_anchors, size_t* bytes) {
  if (!bytes || num_anchors <= 0) return UPSNET_E_BADARG;
  double* pd; int* pi;
  *bytes = ups::rpn_layout(num_anchors, nullptr, &pd, &pi);
  return 0;
}

extern "C" int upsnet_rpn_loss_forward(int num_levels, int A, const int* h, const int* w, const float* const* cls_score,
                                       const float* const* bbox_pred, const int64_t* const* labels,
                                       const long long* label_strides, const float* const* bbox_targets,
                                       const float* const* bbox_inside_weights, const float* const* bbox_outside_weights,
                                       const long long* bbox_strides, float rpn_batch_size, float* cls_loss,
                                       float* bbox_loss, void* workspace, size_t workspace_bytes, void* stream) {
  using namespace ups;
  RpnArgs a{};
  int rc = rpn_args(a, num_levels, A, h, w, cls_score, bbox_pred, labels, label_strides, bbox_targets, bbox_inside_weights,
                    bbox_outside_weights, bbox_strides, rpn_batch_size);
  if (rc) return rc;
  if (!cls_loss || !bbox_loss || !workspace) return UPSNET_E_BADARG;
  double* pd; int* pi;
  if (workspace_bytes < rpn_layout(a.total, workspace, &pd, &pi)) return UPSNET_E_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const int nblocks = tl_blocks(a.total);
  rpn_forward_kernel<<<nblocks, kTlThreads, 0, st>>>(a, pd, pi);
  UPS_CHECK_LAUNCH();
  rpn_finish_kernel<<<1, kTlThreads, 0, st>>>(pd, pi, nblocks, rpn_batch_size, cls_loss, bbox_loss);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_rpn_loss_backward(int num_levels, int A, const int* h, const int* w, const float* const* cls_score,
                                        const float* const* bbox_pred, const int64_t* const* labels,
                                        const long long* label_strides, const float* const* bbox_targets,
                                        const float* const* bbox_inside_weights, const float* const* bbox_outside_weights,
                                        const long long* bbox_strides, float rpn_batch_size, const float* grad_cls,
                                        const float* grad_bbox, float* const* d_cls_score, float* const* d_bbox_pred,
                                        void* stream) {
  using namespace ups;
  RpnArgs a{};
  int rc = rpn_args(a, num_levels, A, h, w, cls_score, bbox_pred, labels, label_strides, bbox_targets, bbox_inside_weights,
                    bbox_outside_weights, bbox_strides, rpn_batch_size);
  if (rc) return rc;
  if (!grad_cls || !grad_bbox || (!d_cls_score && !d_bbox_pred)) return UPSNET_E_BADARG;
  for (int l = 0; l < num_levels; ++l) {
    a.lv[l].dscore = d_cls_score ? d_cls_score[l] : nullptr;
    a.lv[l].dpred = d_bbox_pred ? d_bbox_pred[l] : nullptr;
  }
  rpn_backward_kernel<<<tl_blocks(a.total), kTlThreads, 0, (cudaStream_t)stream>>>(a, grad_cls, grad_bbox);
  UPS_CHECK_LAUNCH();
  return 0;
}

// ---- Mask R-CNN loss ----------------------------------------------------------------------------
extern "C" int upsnet_mask_rcnn_loss_workspace_bytes(int R, int B, long long mask_numel, size_t* bytes) {
  if (!bytes || R <= 0 || B <= 0 || mask_numel < 0) return UPSNET_E_BADARG;
  ups::MrArgs a{};
  a.R = R; a.B = B; a.mask_n = mask_numel;
  double* pd; int* pi;
  *bytes = ups::mr_layout(a, nullptr, &pd, &pi);
  return 0;
}

extern "C" int upsnet_mask_rcnn_loss_forward(const float* cls_score, const int64_t* cls_label, int R, int K,
                                             const float* bbox_pred, const float* bbox_target,
                                             const float* bbox_inside_weight, const float* bbox_outside_weight, int B,
                                             const float* mask_score, const float* mask_target, long long mask_numel,
                                             float* cls_loss, float* bbox_loss, float* mask_loss, float* accuracy,
                                             int* counts, void* workspace, size_t workspace_bytes, void* stream) {
  using namespace ups;
  MrArgs a{};
  int rc = mr_args(a, cls_score, cls_label, R, K, bbox_pred, bbox_target, bbox_inside_weight, bbox_outside_weight, B,
                   mask_score, mask_target, mask_numel);
  if (rc) return rc;
  if (!cls_loss || !bbox_loss || !mask_loss || !accuracy || !counts || !workspace) return UPSNET_E_BADARG;
  double* pd; int* pi;
  if (workspace_bytes < mr_layout(a, workspace, &pd, &pi)) return UPSNET_E_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const int nblocks = a.nb_mask + a.nb_bbox + a.nb_cls;
  mr_forward_kernel<<<nblocks, kTlThreads, 0, st>>>(a, pd, pi);
  UPS_CHECK_LAUNCH();
  mr_finish_kernel<<<1, kTlThreads, 0, st>>>(pd, pi, nblocks, R, cls_loss, bbox_loss, mask_loss, accuracy, counts);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_mask_rcnn_loss_backward(const float* cls_score, const int64_t* cls_label, int R, int K,
                                              const float* bbox_pred, const float* bbox_target,
                                              const float* bbox_inside_weight, const float* bbox_outside_weight, int B,
                                              const float* mask_score, const float* mask_target, long long mask_numel,
                                              const int* counts, const float* grad_cls, const float* grad_bbox,
                                              const float* grad_mask, float* d_cls_score, float* d_bbox_pred,
                                              float* d_mask_score, void* stream) {
  using namespace ups;
  MrArgs a{};
  int rc = mr_args(a, cls_score, cls_label, R, K, bbox_pred, bbox_target, bbox_inside_weight, bbox_outside_weight, B,
                   mask_score, mask_target, mask_numel);
  if (rc) return rc;
  if (!counts || !grad_cls || !grad_bbox || !grad_mask || (!d_cls_score && !d_bbox_pred && !d_mask_score))
    return UPSNET_E_BADARG;
  a.dcls = d_cls_score; a.dpred = d_bbox_pred; a.dmask = mask_numel > 0 ? d_mask_score : nullptr;
  mr_backward_kernel<<<a.nb_mask + a.nb_bbox + a.nb_cls, kTlThreads, 0, (cudaStream_t)stream>>>(a, counts, grad_cls,
                                                                                               grad_bbox, grad_mask);
  UPS_CHECK_LAUNCH();
  return 0;
}

// ---- FCN ROI loss -------------------------------------------------------------------------------
extern "C" int upsnet_fcn_roi_loss_workspace_bytes(int S, int R, int M, int backward, size_t* bytes) {
  if (!bytes || S <= 0 || R < 0 || M <= 0) return UPSNET_E_BADARG;
  if (R == 0 || R > ups::kFrMaxR || M > ups::kFrMaxM) return UPSNET_E_UNSUPPORTED;
  double* pd; int* pi; float* gc; float* corr;
  *bytes = ups::fr_layout(S, R, M, backward, nullptr, &pd, &pi, &gc, &corr);
  return 0;
}

extern "C" int upsnet_fcn_roi_loss_forward(const float* fcn_score, const float* bias, int S, int h, int w, const float* rois,
                                           int R, const void* seg_roi_gt, int seg_roi_gt_is_int64, int M,
                                           int sampling_ratio, float spatial_scale, float* loss, int* counts, float* lse,
                                           void* workspace, size_t workspace_bytes, void* stream) {
  using namespace ups;
  int rc = fr_check(fcn_score, bias, S, h, w, rois, R, seg_roi_gt, M, sampling_ratio, spatial_scale);
  if (rc) return rc;
  if (!loss || !counts || !lse || !workspace) return UPSNET_E_BADARG;
  double* pd; int* pi; float* gc; float* corr;
  if (workspace_bytes < fr_layout(S, R, M, 0, workspace, &pd, &pi, &gc, &corr)) return UPSNET_E_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const int cells = R * M * M, nblocks = tl_blocks(cells);
  if (seg_roi_gt_is_int64)
    fr_forward_kernel<int64_t><<<nblocks, kTlThreads, 0, st>>>(fcn_score, bias, S, h, w, rois, R, M, spatial_scale,
                                                               (const int64_t*)seg_roi_gt, lse, pd, pi);
  else
    fr_forward_kernel<unsigned char><<<nblocks, kTlThreads, 0, st>>>(fcn_score, bias, S, h, w, rois, R, M, spatial_scale,
                                                                     (const unsigned char*)seg_roi_gt, lse, pd, pi);
  UPS_CHECK_LAUNCH();
  fr_finish_kernel<<<1, kTlThreads, 0, st>>>(pd, pi, nblocks, cells, loss, counts);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_fcn_roi_loss_backward(const float* fcn_score, const float* bias, int S, int h, int w, const float* rois,
                                            int R, const void* seg_roi_gt, int seg_roi_gt_is_int64, int M,
                                            int sampling_ratio, float spatial_scale, const float* lse,
                                            const float* grad_out, float* d_fcn_score, float* d_bias, void* workspace,
                                            size_t workspace_bytes, void* stream) {
  using namespace ups;
  int rc = fr_check(fcn_score, bias, S, h, w, rois, R, seg_roi_gt, M, sampling_ratio, spatial_scale);
  if (rc) return rc;
  if (!lse || !grad_out || !d_fcn_score || !d_bias || !workspace) return UPSNET_E_BADARG;
  double* pd; int* pi; float* gc; float* corr;
  if (workspace_bytes < fr_layout(S, R, M, 1, workspace, &pd, &pi, &gc, &corr)) return UPSNET_E_WORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const int cells = R * M * M;
  if (seg_roi_gt_is_int64)
    fr_grad_kernel<int64_t><<<tl_blocks(cells), kTlThreads, 0, st>>>(fcn_score, bias, S, h, w, rois, R, M, spatial_scale,
                                                                     (const int64_t*)seg_roi_gt, lse, grad_out, gc, corr);
  else
    fr_grad_kernel<unsigned char><<<tl_blocks(cells), kTlThreads, 0, st>>>(fcn_score, bias, S, h, w, rois, R, M,
                                                                           spatial_scale, (const unsigned char*)seg_roi_gt,
                                                                           lse, grad_out, gc, corr);
  UPS_CHECK_LAUNCH();
  fr_gather_kernel<<<dim3(tl_blocks((long long)h * w), ceil_div(S, kFrCh)), kTlThreads, 0, st>>>(gc, rois, R, M,
                                                                                                  spatial_scale, S, h, w,
                                                                                                  d_fcn_score);
  UPS_CHECK_LAUNCH();
  fr_dbias_kernel<<<S, kTlThreads, 0, st>>>(gc, corr, cells, d_bias);
  UPS_CHECK_LAUNCH();
  return 0;
}
