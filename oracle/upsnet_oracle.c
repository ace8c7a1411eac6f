/*
 * upsnet_oracle.c -- CPU restatement of the UPSNet per-image inference hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under upsnet_b200/ (the product) may link,
 * import or call this file.  Allowed users: tests/, __graft_entry__.smoke(), and
 * bench.py's cpu_baseline / --impl reference legs.
 *
 * Parity status: the reference ships NO tests / golden vectors for this path
 * (SURVEY.md section 4), so the oracle is pinned against
 *   (i)   the reference's own pure-numpy NMS (upsnet/nms/py_cpu_nms.py), imported
 *         in the build container by tests/golden/make_golden.py -> committed fixtures;
 *   (ii)  the reference's own CUDA kernels compiled for sm_90a (oracle/_ref, built
 *         by oracle/Makefile from the sources where they lie) on the GPU box;
 *   (iii) torchvision.ops.roi_align / deform_conv2d (same Caffe2 / MSRA lineage).
 * The panoptic head's cv2.resize step is NOT bit-reproducible from any formula
 * (SURVEY.md A.5): for that one step the oracle-of-record is the explicit fp32
 * formula below and "parity unpinned" applies to that step (DESIGN.md section 3).
 *
 * Every function cites the reference file:line it restates
 * (paths relative to /root/reference/upsnet/).
 *
 * Build: see oracle/Makefile  (gcc -O2 -fopenmp -ffp-contract=off -shared -fPIC).
 * -ffp-contract=off matters: the panoptic bit-exactness contract is defined on
 * un-fused fp32 multiplies and adds.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORACLE_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------- */
/* ROIAlign forward.  operators/src/roi_align_kernel.cu:43-95 (bilinear),     */
/* :163-235 (RoIAlignForward).  fp32 arithmetic, same operation order.        */
/* ------------------------------------------------------------------------- */
static float roi_bilinear(const float *d, int H, int W, float y, float x) {
  /* roi_align_kernel.cu:51  out-of-range test uses y<-1 || y>H (double compare in
   * the source: -1.0 literal; the comparison result is identical in fp32). */
  if (y < -1.0 || y > H || x < -1.0 || x > W) return 0.f;
  if (y <= 0) y = 0;
  if (x <= 0) x = 0;
  int yl = (int)y, xl = (int)x, yh, xh;
  if (yl >= H - 1) { yh = yl = H - 1; y = (float)yl; } else yh = yl + 1;
  if (xl >= W - 1) { xh = xl = W - 1; x = (float)xl; } else xh = xl + 1;
  float ly = y - yl, lx = x - xl;
  /* roi_align_kernel.cu:83  `1. - ly` is evaluated in double then rounded. */
  float hy = (float)(1. - ly), hx = (float)(1. - lx);
  float v1 = d[yl * W + xl], v2 = d[yl * W + xh], v3 = d[yh * W + xl], v4 = d[yh * W + xh];
  float w1 = hy * hx, w2 = hy * lx, w3 = ly * hx, w4 = ly * lx;
  return (w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4);
}

/* feat: [B,C,H,W] fp32 NCHW; rois: [R,5] (batch,x1,y1,x2,y2); out: [R,C,PH,PW] */
ORACLE_API void oracle_roi_align_forward(const float *feat, int B, int C, int H, int W,
                                         const float *rois, int R, int PH, int PW,
                                         int sampling_ratio, float spatial_scale, float *out) {
  (void)B;
#pragma omp parallel for collapse(2) schedule(static)
  for (int n = 0; n < R; ++n)
    for (int c = 0; c < C; ++c) {
      const float *r = rois + n * 5;
      int b = (int)round(r[0]); /* roi_align_kernel.cu:183 */
      float rsw = r[1] * spatial_scale, rsh = r[2] * spatial_scale;
      float rew = r[3] * spatial_scale, reh = r[4] * spatial_scale;
      float rw = fmaxf(rew - rsw, 1.f), rh = fmaxf(reh - rsh, 1.f);
      float bsh = rh / (float)PH, bsw = rw / (float)PW;
      const float *d = feat + ((size_t)b * C + c) * H * W;
      int gh = sampling_ratio > 0 ? sampling_ratio : (int)ceil(rh / PH);
      int gw = sampling_ratio > 0 ? sampling_ratio : (int)ceil(rw / PW);
      const float count = (float)(gh * gw);
      for (int ph = 0; ph < PH; ++ph)
        for (int pw = 0; pw < PW; ++pw) {
          float acc = 0.f;
          for (int iy = 0; iy < gh; ++iy) {
            const float y = rsh + ph * bsh + (float)(iy + .5f) * bsh / (float)gh;
            for (int ix = 0; ix < gw; ++ix) {
              const float x = rsw + pw * bsw + (float)(ix + .5f) * bsw / (float)gw;
              acc += roi_bilinear(d, H, W, y, x);
            }
          }
          out[(((size_t)n * C + c) * PH + ph) * PW + pw] = acc / count;
        }
    }
}

/* FPN level of a roi.  operators/modules/fpn_roi_align.py:35-38 :
 *   w = x2-x1+1; h = y2-y1+1; k = clip(floor(2 + log2(sqrt(w*h)/224 + 1e-6)), 0, 3)
 * numpy evaluates this in float32 when rois is float32.  Bit-level agreement of
 * log2f between libms is not guaranteed; tests pin this function against numpy
 * itself (tests/test_oracle_cpu.py) and the product uses monotone thresholds. */
ORACLE_API void oracle_fpn_level(const float *rois, int R, int *level) {
  for (int n = 0; n < R; ++n) {
    const float *r = rois + n * 5;
    float w = r[3] - r[1] + 1.f, h = r[4] - r[2] + 1.f;
    float x = sqrtf(w * h) / 224.f + 1e-6f;
    float k = floorf(2.f + log2f(x));
    level[n] = (int)fminf(fmaxf(k, 0.f), 3.f);
  }
}

/* ------------------------------------------------------------------------- */
/* Deformable im2col (v1 / v2).  operators/src/deform_conv_kernel.cu:89-118   */
/* (bilinear), :194-242 (im2col); v2: mod_deform_conv_kernel.cu:187-249.      */
/* ------------------------------------------------------------------------- */
static float dcn_bilinear(const float *d, int H, int W, float h, float w) {
  int hl = (int)floorf(h), wl = (int)floorf(w);
  int hh = hl + 1, wh = wl + 1;
  float lh = h - hl, lw = w - wl, ch = 1 - lh, cw = 1 - lw;
  float v1 = (hl >= 0 && wl >= 0) ? d[hl * W + wl] : 0.f;
  float v2 = (hl >= 0 && wh <= W - 1) ? d[hl * W + wh] : 0.f;
  float v3 = (hh <= H - 1 && wl >= 0) ? d[hh * W + wl] : 0.f;
  float v4 = (hh <= H - 1 && wh <= W - 1) ? d[hh * W + wh] : 0.f;
  float w1 = ch * cw, w2 = ch * lw, w3 = lh * cw, w4 = lh * lw;
  return (w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4);
}

static inline int conv_out(int in, int pad, int dil, int k, int stride) {
  return (in + 2 * pad - (dil * (k - 1) + 1)) / stride + 1;
}

/* One image.  x:[Cin,H,W]  offset:[dg*2*kh*kw,Ho,Wo]  mask:[dg*kh*kw,Ho,Wo] or NULL
 * col:[Cin*kh*kw, Ho*Wo]   (col layout: deform_conv_kernel.cu:212, parallel_imgs=1) */
ORACLE_API void oracle_deform_im2col(const float *x, const float *offset, const float *mask,
                                     int Cin, int H, int W, int kh, int kw, int ph, int pw,
                                     int sh, int sw, int dh, int dw, int dg, float *col) {
  const int Ho = conv_out(H, ph, dh, kh, sh), Wo = conv_out(W, pw, dw, kw, sw);
  const int cpg = Cin / dg;
#pragma omp parallel for schedule(static)
  for (int c = 0; c < Cin; ++c) {
    const int g = c / cpg;
    const float *im = x + (size_t)c * H * W;
    const float *off = offset + (size_t)g * 2 * kh * kw * Ho * Wo;
    const float *msk = mask ? mask + (size_t)g * kh * kw * Ho * Wo : NULL;
    for (int ho = 0; ho < Ho; ++ho)
      for (int wo = 0; wo < Wo; ++wo) {
        const int h_in = ho * sh - ph, w_in = wo * sw - pw;
        for (int i = 0; i < kh; ++i)
          for (int j = 0; j < kw; ++j) {
            const int t = i * kw + j;
            const float oh = off[((size_t)(2 * t) * Ho + ho) * Wo + wo];
            const float ow = off[((size_t)(2 * t + 1) * Ho + ho) * Wo + wo];
            const float him = h_in + i * dh + oh, wim = w_in + j * dw + ow;
            float val = 0.f;
            if (him > -1 && wim > -1 && him < H && wim < W) val = dcn_bilinear(im, H, W, him, wim);
            if (msk) val = val * msk[((size_t)t * Ho + ho) * Wo + wo];
            col[((size_t)(c * kh * kw + t)) * Ho * Wo + (size_t)ho * Wo + wo] = val;
          }
      }
  }
}

/* Full op: im2col + GEMM + bias, per image.  operators/functions/deform_conv.py:44-57
 * (v2: functions/mod_deform_conv.py:44-59).  The reference GEMM is torch.mm fp32 with
 * unspecified summation order; the oracle accumulates in double and rounds once.
 * x:[N,Cin,H,W] offset:[N,dg*2*k*k,Ho,Wo] mask:[N,dg*k*k,Ho,Wo]|NULL
 * weight:[Cout,Cin*kh*kw] bias:[Cout]|NULL  y:[N,Cout,Ho,Wo] */
ORACLE_API int oracle_deform_conv_forward(const float *x, const float *offset, const float *mask,
                                          const float *weight, const float *bias, float *y, int N,
                                          int Cin, int H, int W, int Cout, int kh, int kw, int sh,
                                          int sw, int ph, int pw, int dh, int dw, int dg) {
  const int Ho = conv_out(H, ph, dh, kh, sh), Wo = conv_out(W, pw, dw, kw, sw);
  const int K = Cin * kh * kw;
  const size_t P = (size_t)Ho * Wo;
  float *col = (float *)malloc(sizeof(float) * K * P);
  if (!col) return -1;
  for (int n = 0; n < N; ++n) {
    oracle_deform_im2col(x + (size_t)n * Cin * H * W, offset + (size_t)n * dg * 2 * kh * kw * P,
                         mask ? mask + (size_t)n * dg * kh * kw * P : NULL, Cin, H, W, kh, kw, ph,
                         pw, sh, sw, dh, dw, dg, col);
#pragma omp parallel for schedule(static)
    for (int co = 0; co < Cout; ++co) {
      double *acc = (double *)calloc(P, sizeof(double));
      for (int k = 0; k < K; ++k) {
        const double wv = weight[(size_t)co * K + k];
        const float *cr = col + (size_t)k * P;
        for (size_t p = 0; p < P; ++p) acc[p] += wv * cr[p];
      }
      float *yo = y + ((size_t)n * Cout + co) * P;
      const float b = bias ? bias[co] : 0.f;
      for (size_t p = 0; p < P; ++p) yo[p] = (float)acc[p] + b;
      free(acc);
    }
  }
  free(col);
  return 0;
}

/* ------------------------------------------------------------------------- */
/* NMS.  nms/nms_kernel.cu:30-38 (devIoU, +1 areas), :130-146 (greedy sweep,  */
/* suppress IoU > thresh)  ==  nms/py_cpu_nms.py:16-44.                       */
/* dets:[N,5] (x1,y1,x2,y2,score) in ORIGINAL order; order = argsort desc     */
/* (nms/gpu_nms.pyx:32-33).  Ties in score are unspecified in the reference   */
/* (np.argsort()[::-1] is unstable); the oracle uses stable-desc by index.    */
/* ------------------------------------------------------------------------- */
static float dev_iou(const float *a, const float *b) {
  float left = fmaxf(a[0], b[0]), right = fminf(a[2], b[2]);
  float top = fmaxf(a[1], b[1]), bottom = fminf(a[3], b[3]);
  float width = fmaxf(right - left + 1, 0.f), height = fmaxf(bottom - top + 1, 0.f);
  float interS = width * height;
  float Sa = (a[2] - a[0] + 1) * (a[3] - a[1] + 1);
  float Sb = (b[2] - b[0] + 1) * (b[3] - b[1] + 1);
  return interS / (Sa + Sb - interS);
}

typedef struct { float s; int i; } score_idx;
static int cmp_desc(const void *a, const void *b) {
  const score_idx *x = (const score_idx *)a, *y = (const score_idx *)b;
  if (x->s > y->s) return -1;
  if (x->s < y->s) return 1;
  return x->i - y->i;
}

ORACLE_API void oracle_nms(const float *dets, int N, float thresh, int *keep_out, int *num_out) {
  score_idx *ord = (score_idx *)malloc(sizeof(score_idx) * (N > 0 ? N : 1));
  for (int i = 0; i < N; ++i) { ord[i].s = dets[i * 5 + 4]; ord[i].i = i; }
  qsort(ord, N, sizeof(score_idx), cmp_desc);
  unsigned char *removed = (unsigned char *)calloc(N > 0 ? N : 1, 1);
  int nk = 0;
  for (int i = 0; i < N; ++i) {
    if (removed[i]) continue;
    keep_out[nk++] = ord[i].i;
    const float *a = dets + (size_t)ord[i].i * 5;
    for (int j = i + 1; j < N; ++j)
      if (!removed[j] && dev_iou(a, dets + (size_t)ord[j].i * 5) > thresh) removed[j] = 1;
  }
  *num_out = nk;
  free(removed);
  free(ord);
}

/* ------------------------------------------------------------------------- */
/* Box decode + clip.  bbox/bbox_transform.py:290-330 (bbox_transform),       */
/* :45-60 (clip_boxes).  float32 arithmetic (boxes are cast to deltas.dtype). */
/* boxes:[N,4]  deltas:[N,4*K]  out:[N,4*K]                                   */
/* NOTE np.exp float32 vs expf may differ in the last ulp; tests use 1e-4 tol */
/* on decoded boxes and exact equality only on index outputs downstream.      */
/* ------------------------------------------------------------------------- */
ORACLE_API void oracle_bbox_transform(const float *boxes, const float *deltas, int N, int K,
                                      float wx, float wy, float ww, float wh, float *out) {
  const float clipv = (float)log(1000. / 16.);
  for (int n = 0; n < N; ++n) {
    const float *b = boxes + n * 4;
    float width = b[2] - b[0] + 1.0f, height = b[3] - b[1] + 1.0f;
    float cx = b[0] + 0.5f * width, cy = b[1] + 0.5f * height;
    for (int k = 0; k < K; ++k) {
      const float *d = deltas + ((size_t)n * K + k) * 4;
      float dx = d[0] / wx, dy = d[1] / wy, dw = d[2] / ww, dh = d[3] / wh;
      dw = fminf(dw, clipv);
      dh = fminf(dh, clipv);
      float pcx = dx * width + cx, pcy = dy * height + cy;
      float pw = expf(dw) * width, phh = expf(dh) * height;
      float *o = out + ((size_t)n * K + k) * 4;
      o[0] = pcx - 0.5f * pw;
      o[1] = pcy - 0.5f * phh;
      o[2] = pcx + 0.5f * pw - 1;
      o[3] = pcy + 0.5f * phh - 1;
    }
  }
}

ORACLE_API void oracle_clip_boxes(float *boxes, int N4, float im_h, float im_w) {
  for (int i = 0; i < N4; ++i) {
    float *b = boxes + (size_t)i * 4;
    b[0] = fmaxf(fminf(b[0], im_w - 1), 0.f);
    b[1] = fmaxf(fminf(b[1], im_h - 1), 0.f);
    b[2] = fmaxf(fminf(b[2], im_w - 1), 0.f);
    b[3] = fmaxf(fminf(b[3], im_h - 1), 0.f);
  }
}

/* ------------------------------------------------------------------------- */
/* Panoptic head.  models/resnet_upsnet.py:217-247 with                       */
/*   MaskRemoval  operators/modules/mask_removal.py:29-93                     */
/*   SegTerm      operators/modules/unary_logits.py:78-105                    */
/* The 28x28 -> (w,h) resize (mask_removal.py:68, cv2.resize INTER_LINEAR) is */
/* restated as OpenCV's documented algorithm in un-fused fp32:                */
/*   fx = (float)((dx+0.5)*(28.0/w) - 0.5) [double], sx=floor(fx), fx-=sx;    */
/*   sx<0 -> (0,0);  sx>=27 -> (27,0);   horizontal blend S[sx]*(1-fx)+S[sx+1]*fx */
/*   fy likewise but rows are clamped instead of the fraction (OpenCV resize  */
/*   clips source rows, keeps beta); vertical blend H0*(1-fy)+H1*fy.          */
/* ------------------------------------------------------------------------- */
#define MASK_S 28

static inline void resize_coef_x(int d, int n_dst, int *s_out, float *f_out) {
  double scale = (double)MASK_S / (double)n_dst;
  float f = (float)(((double)d + 0.5) * scale - 0.5);
  int s = (int)floorf(f);
  f = f - (float)s;
  if (s < 0) { s = 0; f = 0.f; }
  if (s >= MASK_S - 1) { s = MASK_S - 1; f = 0.f; }
  *s_out = s;
  *f_out = f;
}
static inline void resize_coef_y(int d, int n_dst, int *s_out, float *f_out) {
  double scale = (double)MASK_S / (double)n_dst;
  float f = (float)(((double)d + 0.5) * scale - 0.5);
  int s = (int)floorf(f);
  f = f - (float)s;
  *s_out = s;
  *f_out = f;
}
static inline int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

/* value of the resized 28x28 logit at box-local integer position (dx,dy), box size (w,h) */
static inline float resized_logit(const float *S, int dx, int dy, int w, int h) {
  int sx, sy;
  float fx, fy;
  resize_coef_x(dx, w, &sx, &fx);
  resize_coef_y(dy, h, &sy, &fy);
  int sx1 = sx + 1 > MASK_S - 1 ? MASK_S - 1 : sx + 1;
  int y0 = clampi(sy, 0, MASK_S - 1), y1 = clampi(sy + 1, 0, MASK_S - 1);
  float a0 = 1.f - fx, a1 = fx, b0 = 1.f - fy, b1 = fy;
  float h0 = S[y0 * MASK_S + sx] * a0 + S[y0 * MASK_S + sx1] * a1;
  float h1 = S[y1 * MASK_S + sx] * a0 + S[y1 * MASK_S + sx1] * a1;
  return h0 * b0 + h1 * b1;
}

/* Resize one 28x28 logit to (w,h): exported so tests can compare with cv2.resize. */
ORACLE_API void oracle_mask_resize(const float *S, int w, int h, float *out) {
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) out[(size_t)y * w + x] = resized_logit(S, x, y, w, h);
}

/* np.round (half to even) on float32, as boxes[i][3].round() in unary_logits.py:100-102 */
static inline float round_half_even(float v) { return nearbyintf(v); }

/*
 * Inputs (one image):
 *   fcn      [S, H, W]  semantic logits (fcn_output), S = num_seg_classes
 *   boxes    [n, 4]     mask_rois[:,1:]  (x1,y1,x2,y2) fp32
 *   cls_prob [n], mask_logit [n,28,28] (logit of the predicted class), cls_idx [n] (1-based thing class)
 *   num_stuff = S - (num_classes-1);  class c -> fcn channel num_stuff + c - 1  (unary_logits.py:72)
 * Outputs:
 *   keep_out [<=n] original indices in score order, *k_out their number (reference quirk: if nothing is
 *   kept, keep=[0] with an all-zero mask plane: mask_removal.py:89-92)
 *   labels [H,W] int64 : argmax over [stuff..., inst 0..k-1, void] with void -> 255 (resnet_upsnet.py:234-240)
 *   sem_labels [H,W] int64 (optional, may be NULL): argmax_c fcn  (resnet_upsnet.py:213)
 * Ties: first max index wins (numpy / torch-CPU argmax convention).
 * Returns 0, or -1 on allocation failure.
 */
ORACLE_API int oracle_panoptic_head(const float *fcn, int S, int H, int W, const float *boxes,
                                    const float *cls_prob, const float *mask_logit,
                                    const int64_t *cls_idx, int n, int num_stuff,
                                    double fraction_threshold, int64_t *keep_out, int *k_out,
                                    int64_t *labels, int64_t *sem_labels) {
  const size_t HW = (size_t)H * W;
  /* ---- MaskRemoval (mask_removal.py:43-93) ---- */
  score_idx *ord = (score_idx *)malloc(sizeof(score_idx) * (n > 0 ? n : 1));
  for (int i = 0; i < n; ++i) { ord[i].s = cls_prob[i]; ord[i].i = i; }
  qsort(ord, n, sizeof(score_idx), cmp_desc); /* np.argsort(cls_prob)[::-1]; ties unspecified */
  int maxc = 0;
  for (int i = 0; i < n; ++i) if (cls_idx[i] > maxc) maxc = (int)cls_idx[i];
  int k = 0;
  int dummy_single = (n == 1 && cls_idx[0] == 0); /* mask_removal.py:55-57 */
  unsigned char *mask_image = NULL; /* [maxc][H][W] uint8 (wraps like numpy uint8 +=) */
  if (!dummy_single && maxc > 0) {
    mask_image = (unsigned char *)calloc((size_t)maxc * HW, 1);
    if (!mask_image) { free(ord); return -1; }
  }
  if (!dummy_single) {
    for (int r = 0; r < n; ++r) {
      const int i = ord[r].i;
      const float *b = boxes + (size_t)i * 4;
      /* ref_boxes = mask_rois.astype(np.int32): truncation toward zero */
      int bx0 = (int)b[0], by0 = (int)b[1], bx1 = (int)b[2], by1 = (int)b[3];
      int w = bx1 - bx0 + 1, h = by1 - by0 + 1;
      if (w < 1) w = 1;
      if (h < 1) h = 1;
      int x0 = bx0 > 0 ? bx0 : 0, x1 = bx1 + 1 < W ? bx1 + 1 : W;
      int y0 = by0 > 0 ? by0 : 0, y1 = by1 + 1 < H ? by1 + 1 : H;
      const int c = (int)cls_idx[i] - 1;
      const float *Sm = mask_logit + (size_t)i * MASK_S * MASK_S;
      long mask_sum = 0, overlap = 0;
      unsigned char *mi = (c >= 0) ? mask_image + (size_t)c * HW : NULL;
      /* crop_mask indices beyond the (w,h) logit are empty slices in numpy */
      for (int y = y0; y < y1; ++y) {
        int dy = y - by0;
        if (dy < 0 || dy >= h) continue;
        for (int x = x0; x < x1; ++x) {
          int dx = x - bx0;
          if (dx < 0 || dx >= w) continue;
          if (resized_logit(Sm, dx, dy, w, h) > 0) {
            ++mask_sum;
            if (mi && mi[(size_t)y * W + x] >= 1) ++overlap;
          }
        }
      }
      if (mask_sum == 0 || ((double)overlap / (double)mask_sum > fraction_threshold)) continue;
      keep_out[k++] = i;
      if (mi)
        for (int y = y0; y < y1; ++y) {
          int dy = y - by0;
          if (dy < 0 || dy >= h) continue;
          for (int x = x0; x < x1; ++x) {
            int dx = x - bx0;
            if (dx < 0 || dx >= w) continue;
            if (resized_logit(Sm, dx, dy, w, h) > 0) mi[(size_t)y * W + x] += 1;
          }
        }
    }
  }
  free(mask_image);
  int zero_mask = 0; /* reference fallback: keep=[0], mask_energy = zeros [1,1,H,W] */
  if (k == 0) { keep_out[0] = 0; k = 1; zero_mask = 1; }
  *k_out = k;

  /* ---- per kept instance geometry ---- */
  int *geo = (int *)malloc(sizeof(int) * (size_t)k * 12);
  if (!geo) { free(ord); return -1; }
  int *gx0 = geo, *gy0 = geo + k, *gx1 = geo + 2 * k, *gy1 = geo + 3 * k; /* mask paste window */
  int *bx0s = geo + 4 * k, *by0s = geo + 5 * k, *ws = geo + 6 * k, *hs = geo + 7 * k; /* int box */
  int *sx0 = geo + 8 * k, *sy0 = geo + 9 * k, *sx1 = geo + 10 * k, *sy1 = geo + 11 * k; /* SegTerm window */
  for (int j = 0; j < k; ++j) {
    const int i = (int)keep_out[j];
    const float *b = boxes + (size_t)i * 4;
    int bx0 = (int)b[0], by0 = (int)b[1], bx1 = (int)b[2], by1 = (int)b[3];
    int w = bx1 - bx0 + 1, h = by1 - by0 + 1;
    if (w < 1) w = 1;
    if (h < 1) h = 1;
    bx0s[j] = bx0; by0s[j] = by0; ws[j] = w; hs[j] = h;
    gx0[j] = bx0 > 0 ? bx0 : 0; gx1[j] = bx1 + 1 < W ? bx1 + 1 : W;
    gy0[j] = by0 > 0 ? by0 : 0; gy1[j] = by1 + 1 < H ? by1 + 1 : H;
    /* SegTerm window (unary_logits.py:92-103): boxes*4*(1/4) is exact; y0=int(b1), y1=int(round(b3)+1) */
    float fb0 = b[0] * 4.0f * 0.25f, fb1 = b[1] * 4.0f * 0.25f, fb2 = b[2] * 4.0f * 0.25f, fb3 = b[3] * 4.0f * 0.25f;
    sx0[j] = (int)fb0; sy0[j] = (int)fb1;
    sx1[j] = (int)(round_half_even(fb2) + 1); sy1[j] = (int)(round_half_even(fb3) + 1);
    /* python slice clamping */
    if (sx0[j] > W) sx0[j] = W;
    if (sy0[j] > H) sy0[j] = H;
    if (sx1[j] > W) sx1[j] = W;
    if (sy1[j] > H) sy1[j] = H;
    if (cls_idx[i] == 0) { sx1[j] = sx0[j]; sy1[j] = sy0[j]; } /* unary_logits.py:97-98: skipped -> zeros */
  }

  /* ---- fused per-pixel argmax (resnet_upsnet.py:234-240) ---- */
#pragma omp parallel for schedule(static)
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      const size_t p = (size_t)y * W + x;
      float best = fcn[p];
      int bi = 0;
      float sem_best = fcn[p];
      int sem_bi = 0;
      for (int c = 1; c < S; ++c) {
        float v = fcn[(size_t)c * HW + p];
        if (c < num_stuff && v > best) { best = v; bi = c; }
        if (v > sem_best) { sem_best = v; sem_bi = c; }
      }
      float thing_max = fcn[(size_t)num_stuff * HW + p];
      for (int c = num_stuff + 1; c < S; ++c) thing_max = fmaxf(thing_max, fcn[(size_t)c * HW + p]);
      float inst_max = 0.f;
      int inst_max_init = 0;
      for (int j = 0; j < k; ++j) {
        const int i = (int)keep_out[j];
        float seg = 0.f;
        if (x >= sx0[j] && x < sx1[j] && y >= sy0[j] && y < sy1[j])
          seg = fcn[(size_t)(num_stuff + (int)cls_idx[i] - 1) * HW + p];
        float m = 0.f;
        if (!zero_mask && x >= gx0[j] && x < gx1[j] && y >= gy0[j] && y < gy1[j]) {
          int dx = x - bx0s[j], dy = y - by0s[j];
          if (dx >= 0 && dx < ws[j] && dy >= 0 && dy < hs[j])
            m = resized_logit(mask_logit + (size_t)i * MASK_S * MASK_S, dx, dy, ws[j], hs[j]);
        }
        float v = seg + m;
        if (v > best) { best = v; bi = num_stuff + j; }
        if (!inst_max_init) { inst_max = seg; inst_max_init = 1; } else inst_max = fmaxf(inst_max, seg);
      }
      float voidv = thing_max - inst_max;
      if (voidv > best) { best = voidv; bi = num_stuff + k; }
      labels[p] = (bi == num_stuff + k) ? 255 : bi;
      if (sem_labels) sem_labels[p] = sem_bi;
    }
  free(geo);
  free(ord);
  return 0;
}

/* ------------------------------------------------------------------------- */
/* Dense conv2d (NCHW fp32, groups=1) with optional bias/ReLU -- the oracle   */
/* for the backbone/FPN/RPN/head convolutions.  Reference = torch.nn.Conv2d   */
/* (models/resnet.py:80-100 etc., cuDNN); double accumulation, rounded once.  */
/* ------------------------------------------------------------------------- */
ORACLE_API void oracle_conv2d(const float *x, const float *weight, const float *bias, float *y,
                              int N, int Cin, int H, int W, int Cout, int kh, int kw, int sh,
                              int sw, int ph, int pw, int dh, int dw, int relu) {
  const int Ho = conv_out(H, ph, dh, kh, sh), Wo = conv_out(W, pw, dw, kw, sw);
#pragma omp parallel for collapse(2) schedule(static)
  for (int n = 0; n < N; ++n)
    for (int co = 0; co < Cout; ++co)
      for (int ho = 0; ho < Ho; ++ho)
        for (int wo = 0; wo < Wo; ++wo) {
          double acc = 0.0;
          for (int c = 0; c < Cin; ++c)
            for (int i = 0; i < kh; ++i) {
              int hi = ho * sh - ph + i * dh;
              if (hi < 0 || hi >= H) continue;
              for (int j = 0; j < kw; ++j) {
                int wi = wo * sw - pw + j * dw;
                if (wi < 0 || wi >= W) continue;
                acc += (double)x[(((size_t)n * Cin + c) * H + hi) * W + wi] *
                       (double)weight[(((size_t)co * Cin + c) * kh + i) * kw + j];
              }
            }
          float v = (float)acc + (bias ? bias[co] : 0.f);
          if (relu && v < 0.f) v = 0.f;
          y[(((size_t)n * Cout + co) * Ho + ho) * Wo + wo] = v;
        }
}
