// upsample2.cu -- the FPN top-down path's bilinear 2x up-sampling on NHWC activations (models/fpn.py:27-35 with
// network.fpn_upsample_method = 'bilinear': F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=False))
// and its adjoint.  The rule is bilin.cuh's.
//
// Forward: one thread = one output pixel x 8 channels: four 16-byte (bf16) or 32-byte (fp32, hi/lo pair) corner reads,
// interpolated in fp32 (a pair's value is hi + lo) and rounded once to the output format.  The four corners of
// neighbouring output pixels overlap, so L1/L2 serve them and HBM sees the coarse map about once (roofline: HBM, the
// coarse map in and the 4x larger fine map out).
// Adjoint: a gather, one thread = one coarse pixel x 4 channels: the sum of its 4x4 fine footprint (rows / columns
// 2s - 1 .. 2s + 2 inside the map) with the weights bilin_tap gives them, along x per row and then along y, in a fixed
// order.  No atomics: the same input gives the same bytes.
#include <cuda_bf16.h>

#include "bilin.cuh"
#include "common.cuh"
#include "pair.cuh"

namespace ups {
namespace {

// eight channels (16-byte unit cv of the C / 8 per pixel) of pixel `pix` of an NHWC map with C8 = C / 8
template <int DT>
__device__ __forceinline__ void load8(const uint4* __restrict__ x, size_t pix, int C8, int cv, float* v) {
  if (DT == UPSNET_DTYPE_BF16) {
    const uint4 a = __ldg(x + pix * C8 + cv);
    const uint32_t u[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      v[2 * e] = bf16x2_x(u[e]);
      v[2 * e + 1] = bf16x2_y(u[e]);
    }
  } else if (DT == UPSNET_DTYPE_PAIR) {
    const uint4 h = __ldg(x + pix * 2 * C8 + cv), l = __ldg(x + pix * 2 * C8 + C8 + cv);
    const uint32_t hu[4] = {h.x, h.y, h.z, h.w}, lu[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      v[2 * e] = pair_x(hu[e], lu[e]);
      v[2 * e + 1] = pair_y(hu[e], lu[e]);
    }
  } else {
    const float4 a = __ldg(reinterpret_cast<const float4*>(x) + pix * 2 * C8 + 2 * cv);
    const float4 b = __ldg(reinterpret_cast<const float4*>(x) + pix * 2 * C8 + 2 * cv + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  }
}

template <int DT>
__device__ __forceinline__ void store8(uint4* __restrict__ y, size_t pix, int C8, int cv, const float* o) {
  if (DT == UPSNET_DTYPE_BF16) {
    y[pix * C8 + cv] = pack_bf16x8(o);
  } else if (DT == UPSNET_DTYPE_PAIR) {
    uint4 hi, lo;
    split_pair8(o, hi, lo);
    y[pix * 2 * C8 + cv] = hi;
    y[pix * 2 * C8 + C8 + cv] = lo;
  } else {
    float4* f = reinterpret_cast<float4*>(y) + pix * 2 * C8 + 2 * cv;
    f[0] = make_float4(o[0], o[1], o[2], o[3]);
    f[1] = make_float4(o[4], o[5], o[6], o[7]);
  }
}

template <int DT>
__global__ void __launch_bounds__(256)
up2_bilinear_nhwc_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, int N, int h, int w, int C8) {
  const int H = 2 * h, W = 2 * w;
  const long long total = (long long)N * H * W * C8;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(t % C8);
    const long long pix = t / C8;
    const int xo = (int)(pix % W), yo = (int)(pix / W % H);
    const size_t n = (size_t)(pix / ((long long)W * H));
    const BilinAxis ay = bilin_axis(yo, h, 2), ax = bilin_axis(xo, w, 2);
    const size_t r0 = (n * h + ay.i0) * w, r1 = (n * h + ay.i1) * w;
    float a[8], b[8], c[8], d[8], o[8];
    load8<DT>(x, r0 + ax.i0, C8, cv, a);
    load8<DT>(x, r0 + ax.i1, C8, cv, b);
    load8<DT>(x, r1 + ax.i0, C8, cv, c);
    load8<DT>(x, r1 + ax.i1, C8, cv, d);
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = bilin_mix(ay, ax, a[e], b[e], c[e], d[e]);
    store8<DT>(y, (size_t)pix, C8, cv, o);
  }
}

__global__ void __launch_bounds__(256)
up2_bilinear_adjoint_kernel(const float4* __restrict__ g, const float4* __restrict__ ymask, float4* __restrict__ d,
                            int N, int h, int w, int C4) {
  const int H = 2 * h, W = 2 * w;
  const long long total = (long long)N * h * w * C4;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(t % C4);
    const long long q = t / C4;
    const int xs = (int)(q % w), ys = (int)(q / w % h);
    const size_t n = (size_t)(q / ((long long)w * h));
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int ky = 0; ky < 4; ++ky) {
      const int oy = 2 * ys - 1 + ky;
      if (oy < 0 || oy >= H) continue;
      float row[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int kx = 0; kx < 4; ++kx) {
        const int ox = 2 * xs - 1 + kx;
        if (ox < 0 || ox >= W) continue;
        const float wx = bilin_tap(ox, xs, w, 2);
        const size_t i = ((n * H + oy) * W + ox) * C4 + cv;
        float4 v = __ldg(g + i);
        if (ymask) {       // the ReLU mask of the forward: dz = dy where y > 0
          const float4 yv = __ldg(ymask + i);
          v = make_float4(yv.x > 0.f ? v.x : 0.f, yv.y > 0.f ? v.y : 0.f, yv.z > 0.f ? v.z : 0.f, yv.w > 0.f ? v.w : 0.f);
        }
        row[0] = __fmaf_rn(wx, v.x, row[0]);
        row[1] = __fmaf_rn(wx, v.y, row[1]);
        row[2] = __fmaf_rn(wx, v.z, row[2]);
        row[3] = __fmaf_rn(wx, v.w, row[3]);
      }
      const float wy = bilin_tap(oy, ys, h, 2);
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[e] = __fmaf_rn(wy, row[e], acc[e]);
    }
    d[t] = make_float4(acc[0], acc[1], acc[2], acc[3]);
  }
}

unsigned grid_for(long long total) {
  long long blocks = (total + 255) / 256;
  if (blocks > (long long)num_sms() * 32) blocks = (long long)num_sms() * 32;
  return (unsigned)blocks;
}

}  // namespace

int up2_bilinear_adjoint_launch(const float* dy, const float* ymask, float* dx, int N, int h, int w, int C,
                                cudaStream_t stream) {
  const long long total = (long long)N * h * w * (C / 4);
  up2_bilinear_adjoint_kernel<<<grid_for(total), 256, 0, stream>>>(
      reinterpret_cast<const float4*>(dy), reinterpret_cast<const float4*>(ymask), reinterpret_cast<float4*>(dx), N,
      h, w, C / 4);
  UPS_CHECK_LAUNCH();
  return 0;
}

}  // namespace ups

extern "C" int upsnet_upsample2_bilinear_nhwc(const void* x, void* y, int N, int h, int w, int C, int dtype,
                                              void* stream) {
  using namespace ups;
  if (!x || !y || N <= 0 || h <= 0 || w <= 0 || C <= 0) return UPSNET_E_BADARG;
  if (dtype != UPSNET_DTYPE_F32 && dtype != UPSNET_DTYPE_BF16 && dtype != UPSNET_DTYPE_PAIR) return UPSNET_E_BADARG;
  if (C % 8 || (((uintptr_t)x) & 15) || (((uintptr_t)y) & 15)) return UPSNET_E_UNSUPPORTED;
  const long long total = (long long)N * 2 * h * 2 * w * (C / 8);
  const unsigned blocks = grid_for(total);
  cudaStream_t s = (cudaStream_t)stream;
  const uint4* xi = static_cast<const uint4*>(x);
  uint4* yo = static_cast<uint4*>(y);
  if (dtype == UPSNET_DTYPE_PAIR)
    up2_bilinear_nhwc_kernel<UPSNET_DTYPE_PAIR><<<blocks, 256, 0, s>>>(xi, yo, N, h, w, C / 8);
  else if (dtype == UPSNET_DTYPE_BF16)
    up2_bilinear_nhwc_kernel<UPSNET_DTYPE_BF16><<<blocks, 256, 0, s>>>(xi, yo, N, h, w, C / 8);
  else
    up2_bilinear_nhwc_kernel<UPSNET_DTYPE_F32><<<blocks, 256, 0, s>>>(xi, yo, N, h, w, C / 8);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_upsample2_bilinear_nhwc_adjoint(const float* dy, float* dx, int N, int h, int w, int C,
                                                      void* stream) {
  using namespace ups;
  if (!dy || !dx || N <= 0 || h <= 0 || w <= 0 || C <= 0) return UPSNET_E_BADARG;
  if (C % 4 || (((uintptr_t)dy) & 15) || (((uintptr_t)dx) & 15)) return UPSNET_E_UNSUPPORTED;
  return up2_bilinear_adjoint_launch(dy, nullptr, dx, N, h, w, C, (cudaStream_t)stream);
}
