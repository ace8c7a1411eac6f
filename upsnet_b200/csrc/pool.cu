// pool.cu -- k x k / stride s max-pooling on NHWC activations (the ResNet stem's 3x3/2 pool, models/resnet.py:163
// `self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)`), bf16 or fp32 storage.
// One thread = one output pixel x 8 (bf16) / 4 (fp32) channels: k*k 16-byte reads, one 16-byte write; the
// overlapping windows are served by L1/L2, HBM sees the input once (roofline: HBM, in + out bytes).
#include <cuda_bf16.h>
#include <cfloat>

#include "bilin.cuh"
#include "common.cuh"
#include "pair.cuh"
#include "up4.cuh"

namespace ups {

template <bool BF16>
__global__ void maxpool_nhwc_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int N, int H, int W, int CV,
                                    int Ho, int Wo, int k, int s, int pad) {
  const long long total = (long long)N * Ho * Wo * CV;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(t % CV);
    long long pix = t / CV;
    const int wo = (int)(pix % Wo);
    pix /= Wo;
    const int ho = (int)(pix % Ho), n = (int)(pix / Ho);
    const int h0 = ho * s - pad, w0 = wo * s - pad;
    uint4 best;
    if (BF16) best = make_uint4(0xff80ff80u, 0xff80ff80u, 0xff80ff80u, 0xff80ff80u);     // -inf pairs
    else best = make_uint4(0xff800000u, 0xff800000u, 0xff800000u, 0xff800000u);
    for (int i = 0; i < k; ++i) {
      const int h = h0 + i;
      if (h < 0 || h >= H) continue;
      for (int j = 0; j < k; ++j) {
        const int w = w0 + j;
        if (w < 0 || w >= W) continue;
        const uint4 v = __ldg(x + (((size_t)n * H + h) * W + w) * CV + cv);
        if (BF16) {
          __nv_bfloat162* b = reinterpret_cast<__nv_bfloat162*>(&best);
          const __nv_bfloat162* a = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
          for (int e = 0; e < 4; ++e) b[e] = __hmax2(b[e], a[e]);
        } else {
          float* b = reinterpret_cast<float*>(&best);
          const float* a = reinterpret_cast<const float*>(&v);
#pragma unroll
          for (int e = 0; e < 4; ++e) b[e] = fmaxf(b[e], a[e]);
        }
      }
    }
    y[t] = best;
  }
}

// hi/lo pair storage ([N,H,W,2C] bf16: C hi values then C lo values per pixel): the window element with the largest
// hi + lo (exact in fp32) is copied as it is -- both halves -- so the result is again a canonical pair.
__global__ void maxpool_nhwc_pair_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int N, int H, int W, int CV,
                                         int Ho, int Wo, int k, int s, int pad) {
  const long long total = (long long)N * Ho * Wo * CV;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(t % CV);
    long long pix = t / CV;
    const int wo = (int)(pix % Wo);
    pix /= Wo;
    const int ho = (int)(pix % Ho), n = (int)(pix / Ho);
    const int h0 = ho * s - pad, w0 = wo * s - pad;
    float best[8];
    uint32_t bh[4], bl[4];
#pragma unroll
    for (int e = 0; e < 8; ++e) best[e] = -INFINITY;
#pragma unroll
    for (int e = 0; e < 4; ++e) { bh[e] = 0xff80ff80u; bl[e] = 0u; }
    for (int i = 0; i < k; ++i) {
      const int h = h0 + i;
      if (h < 0 || h >= H) continue;
      for (int j = 0; j < k; ++j) {
        const int w = w0 + j;
        if (w < 0 || w >= W) continue;
        const size_t base = (((size_t)n * H + h) * W + w) * (size_t)(2 * CV);
        const uint4 vh = __ldg(x + base + cv), vl = __ldg(x + base + CV + cv);
        const uint32_t hw[4] = {vh.x, vh.y, vh.z, vh.w}, lw[4] = {vl.x, vl.y, vl.z, vl.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float a = pair_x(hw[e], lw[e]), b = pair_y(hw[e], lw[e]);
          if (a > best[2 * e]) { best[2 * e] = a; bh[e] = (bh[e] & 0xffff0000u) | (hw[e] & 0xffffu); bl[e] = (bl[e] & 0xffff0000u) | (lw[e] & 0xffffu); }
          if (b > best[2 * e + 1]) { best[2 * e + 1] = b; bh[e] = (bh[e] & 0xffffu) | (hw[e] & 0xffff0000u); bl[e] = (bl[e] & 0xffffu) | (lw[e] & 0xffff0000u); }
        }
      }
    }
    const size_t ob = (size_t)(t / CV) * (size_t)(2 * CV);
    y[ob + cv] = make_uint4(bh[0], bh[1], bh[2], bh[3]);
    y[ob + CV + cv] = make_uint4(bl[0], bl[1], bl[2], bl[3]);
  }
}

}  // namespace ups

extern "C" int upsnet_maxpool2d_nhwc(const void* x, void* y, int N, int H, int W, int C, int k, int stride, int pad,
                                     int dtype, void* stream) {
  if (!x || !y || N <= 0 || H <= 0 || W <= 0 || C <= 0 || k <= 0 || stride <= 0 || pad < 0 || 2 * pad > k) return UPSNET_E_BADARG;
  const int vec = dtype == UPSNET_DTYPE_F32 ? 4 : 8;
  if (dtype != UPSNET_DTYPE_BF16 && dtype != UPSNET_DTYPE_F32 && dtype != UPSNET_DTYPE_PAIR) return UPSNET_E_BADARG;
  if (C % vec || (((uintptr_t)x) & 15) || (((uintptr_t)y) & 15)) return UPSNET_E_UNSUPPORTED;
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  if (Ho <= 0 || Wo <= 0) return UPSNET_E_BADARG;
  const long long total = (long long)N * Ho * Wo * (C / vec);
  long long blocks = (total + 255) / 256;
  if (blocks > ups::kNumSMs * 32) blocks = ups::kNumSMs * 32;
  if (dtype == UPSNET_DTYPE_PAIR)
    ups::maxpool_nhwc_pair_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
        (const uint4*)x, (uint4*)y, N, H, W, C / vec, Ho, Wo, k, stride, pad);
  else if (dtype == UPSNET_DTYPE_BF16)
    ups::maxpool_nhwc_kernel<true><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
        (const uint4*)x, (uint4*)y, N, H, W, C / vec, Ho, Wo, k, stride, pad);
  else
    ups::maxpool_nhwc_kernel<false><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
        (const uint4*)x, (uint4*)y, N, H, W, C / vec, Ho, Wo, k, stride, pad);
  UPS_CHECK_LAUNCH();
  return 0;
}

// ----------------------------------------------------------------------------------------------
// Bilinear up-sampling by an integer factor on NCHW fp32 planes, align_corners = False
// (models/fcn.py:88-101 nn.Upsample(scale_factor, mode='bilinear') of the semantic logits).
// src = (dst + 0.5) / f - 0.5 clamped at 0 (the same source-index rule as ATen's upsample_bilinear2d);
// one thread = 4 consecutive output pixels of one row (float4 store).  Roofline: HBM, 4*P*Ho*Wo bytes written.
// ----------------------------------------------------------------------------------------------
namespace ups {

__global__ void __launch_bounds__(256)
upsample_bilinear_nchw_kernel(const float* __restrict__ x, float* __restrict__ y, int P, int H, int W, int f) {
  const int Ho = H * f, Wo = W * f, Wq = Wo >> 2;
  const long long total = (long long)P * Ho * Wq;
  const float rf = 1.0f / (float)f;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int xq = (int)(t % Wq);
    long long rest = t / Wq;
    const int yo = (int)(rest % Ho);
    const int pl = (int)(rest / Ho);
    float o[4];
    if (f == 4) {      // shared with the fused panoptic head (up4.cuh): six loads per quad, explicit FMAs
      const Up4Row rw = up4_row(yo, H);
      up4_quad(x + ((size_t)pl * H + rw.y0) * W, x + ((size_t)pl * H + rw.y1) * W, xq, W, rw.ly, rw.hy, o);
      reinterpret_cast<float4*>(y)[t] = make_float4(o[0], o[1], o[2], o[3]);
      continue;
    }
    const float sy = fmaxf(rf * ((float)yo + 0.5f) - 0.5f, 0.f);
    const int y0 = (int)sy, y1 = y0 + (y0 < H - 1 ? 1 : 0);
    const float ly = sy - (float)y0, hy = 1.f - ly;
    const float* r0 = x + ((size_t)pl * H + y0) * W;
    const float* r1 = x + ((size_t)pl * H + y1) * W;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int xo = xq * 4 + e;
      const float sx = fmaxf(rf * ((float)xo + 0.5f) - 0.5f, 0.f);
      const int x0 = (int)sx, x1 = x0 + (x0 < W - 1 ? 1 : 0);
      const float lx = sx - (float)x0, hx = 1.f - lx;
      o[e] = hy * (hx * __ldg(r0 + x0) + lx * __ldg(r0 + x1)) + ly * (hx * __ldg(r1 + x0) + lx * __ldg(r1 + x1));
    }
    reinterpret_cast<float4*>(y)[t] = make_float4(o[0], o[1], o[2], o[3]);
  }
}

}  // namespace ups

// score = s2 + up2(s3) + up4(s4) + up8(s5): the semantic head's per-level score maps (the 1x1 score conv commutes with the
// bilinear up-sampling, models/fcn.py:94-101) summed at P2 resolution in one pass, same bilinear rule and the same order
// of the three additions as the torch expression it replaces (F.interpolate + add, three times).
namespace ups {
__global__ void __launch_bounds__(256)
fcn_score_fuse_kernel(const float* __restrict__ s2, const float* __restrict__ s3, const float* __restrict__ s4,
                      const float* __restrict__ s5, float* __restrict__ out, int P, int H, int W) {
  const long long total = (long long)P * H * W;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(t % W);
    const long long r = t / W;
    const int y = (int)(r % H), pl = (int)(r / H);
    float v = s2[t];
    v = v + bilin_at(s3 + (size_t)pl * (H / 2) * (W / 2), H / 2, W / 2, 2, y, x);
    v = v + bilin_at(s4 + (size_t)pl * (H / 4) * (W / 4), H / 4, W / 4, 4, y, x);
    v = v + bilin_at(s5 + (size_t)pl * (H / 8) * (W / 8), H / 8, W / 8, 8, y, x);
    out[t] = v;
  }
}
}  // namespace ups

extern "C" int upsnet_fcn_score_fuse(const float* s2, const float* s3, const float* s4, const float* s5, float* out,
                                     int planes, int H, int W, void* stream) {
  if (!s2 || !s3 || !s4 || !s5 || !out || planes <= 0 || H <= 0 || W <= 0) return UPSNET_E_BADARG;
  if ((H & 7) || (W & 7)) return UPSNET_E_UNSUPPORTED;
  const long long total = (long long)planes * H * W;
  long long blocks = (total + 255) / 256;
  if (blocks > ups::kNumSMs * 32) blocks = ups::kNumSMs * 32;
  ups::fcn_score_fuse_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(s2, s3, s4, s5, out, planes, H, W);
  UPS_CHECK_LAUNCH();
  return 0;
}

// The adjoint of fcn_score_fuse: ds_l = up_f^T(dscore) for f = 2, 4, 8 (ds2 is dscore itself).  A gather: every source
// pixel sums its own output footprint, so there are no atomics.  Source index s along an axis receives from the 2f
// output coordinates f s - f/2 .. f s + 3f/2 - 1 (the forward's rule: clamped at 0 below, the last sample repeated
// above), with the weights bilin_at gives it.  One CTA = a kFbTy x kFbTx source tile of one level and one plane:
// A sums along x for every output row of the tile's footprint into shared memory, B sums those rows along y, each in a
// fixed tap order.
namespace ups {
constexpr int kFbTx = 32, kFbTy = 8, kFbThreads = kFbTx * kFbTy;
constexpr int kFbRows = 8 * kFbTy + 8;       // output rows of the x8 footprint of one tile, the largest

__global__ void __launch_bounds__(kFbThreads)
fcn_score_fuse_backward_kernel(const float* __restrict__ g, float* __restrict__ d3, float* __restrict__ d4,
                               float* __restrict__ d5, int H, int W, int tiles3, int tiles4) {
  __shared__ float s_xr[kFbRows * kFbTx];
  int tile = blockIdx.x, lv = 1;
  if (tile >= tiles3 + tiles4) { lv = 3; tile -= tiles3 + tiles4; }
  else if (tile >= tiles3) { lv = 2; tile -= tiles3; }
  const int f = 1 << lv, half = f >> 1, h = H >> lv, w = W >> lv;
  const int tx = (w + kFbTx - 1) / kFbTx;
  const int x0 = (tile % tx) * kFbTx, y0 = (tile / tx) * kFbTy;
  const float* gp = g + (size_t)blockIdx.y * H * W;
  float* dp = (lv == 1 ? d3 : lv == 2 ? d4 : d5) + (size_t)blockIdx.y * h * w;
  const int rows = f * kFbTy + f, oy0 = f * y0 - half;
  // A: output row oy0 + r, source column x0 + bx
  for (int e = threadIdx.x; e < rows * kFbTx; e += kFbThreads) {
    const int r = e / kFbTx, bx = e - r * kFbTx, xs = x0 + bx, oy = oy0 + r;
    float acc = 0.f;
    if (xs < w && oy >= 0 && oy < H) {
      const float* row = gp + (size_t)oy * W;
      for (int k = 0; k < 2 * f; ++k) {
        const int ox = f * xs - half + k;
        if (ox < 0 || ox >= W) continue;
        acc = __fmaf_rn(bilin_tap(ox, xs, w, f), __ldg(row + ox), acc);
      }
    }
    s_xr[e] = acc;
  }
  __syncthreads();
  // B: one source pixel per thread; its output rows are halo rows f * sy .. f * sy + 2f - 1
  const int sx = threadIdx.x % kFbTx, sy = threadIdx.x / kFbTx;
  const int x = x0 + sx, y = y0 + sy;
  if (x < w && y < h) {
    float acc = 0.f;
    for (int k = 0; k < 2 * f; ++k) {
      const int oy = f * y - half + k;
      if (oy < 0 || oy >= H) continue;
      acc = __fmaf_rn(bilin_tap(oy, y, h, f), s_xr[(f * sy + k) * kFbTx + sx], acc);
    }
    dp[(size_t)y * w + x] = acc;
  }
}
}  // namespace ups

extern "C" int upsnet_fcn_score_fuse_backward(const float* dscore, float* ds3, float* ds4, float* ds5, int planes, int H,
                                              int W, void* stream) {
  if (!dscore || !ds3 || !ds4 || !ds5 || planes <= 0 || H <= 0 || W <= 0) return UPSNET_E_BADARG;
  if ((H & 7) || (W & 7) || planes > 65535) return UPSNET_E_UNSUPPORTED;
  long long tiles[3];
  for (int lv = 1; lv <= 3; ++lv)
    tiles[lv - 1] = (long long)ups::ceil_div(W >> lv, ups::kFbTx) * ups::ceil_div(H >> lv, ups::kFbTy);
  const long long total = tiles[0] + tiles[1] + tiles[2];
  if (total > 0x7fffffffLL) return UPSNET_E_UNSUPPORTED;
  ups::fcn_score_fuse_backward_kernel<<<dim3((unsigned)total, (unsigned)planes), ups::kFbThreads, 0, (cudaStream_t)stream>>>(
      dscore, ds3, ds4, ds5, H, W, (int)tiles[0], (int)tiles[1]);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_upsample_bilinear_nchw(const float* x, float* y, int planes, int H, int W, int factor, void* stream) {
  if (!x || !y || planes <= 0 || H <= 0 || W <= 0 || factor <= 0) return UPSNET_E_BADARG;
  if (((W * factor) & 3) || (((uintptr_t)y) & 15)) return UPSNET_E_UNSUPPORTED;
  const long long total = (long long)planes * H * factor * ((W * factor) >> 2);
  long long blocks = (total + 255) / 256;
  if (blocks > ups::kNumSMs * 32) blocks = ups::kNumSMs * 32;
  ups::upsample_bilinear_nchw_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, y, planes, H, W, factor);
  UPS_CHECK_LAUNCH();
  return 0;
}
