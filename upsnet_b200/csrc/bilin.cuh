// bilin.cuh -- the bilinear up-sampling rule of ATen's upsample_bilinear2d with align_corners = False, written down once.
//
// Output coordinate o of an axis of n source samples up-sampled by an integer factor f reads the source position
// src = max((o + 0.5) / f - 0.5, 0): samples i0 = floor(src) and i1 = i0 + 1 (i0 itself on the last sample, so the last
// row / column repeats) with weights h = 1 - l and l = src - i0.  A 2-D value is hy (hx a + lx b) + ly (hx c + lx d) over
// the corners a = (y0, x0), b = (y0, x1), c = (y1, x0), d = (y1, x1).  Every kernel that up-samples bilinearly (the
// semantic head's score sum and its adjoint, the FPN top-down path and its adjoint, the GroupNorm apply's residual)
// forms its taps and its blend through the functions below.
#pragma once
#include <cuda_runtime.h>

namespace ups {

struct BilinAxis {
  int i0, i1;
  float l, h;
};

__device__ __forceinline__ BilinAxis bilin_axis(int o, int n, int f) {
  const float src = fmaxf((1.0f / (float)f) * ((float)o + 0.5f) - 0.5f, 0.f);
  BilinAxis a;
  a.i0 = (int)src;
  a.i1 = a.i0 + (a.i0 < n - 1 ? 1 : 0);
  a.l = src - (float)a.i0;
  a.h = 1.f - a.l;
  return a;
}

__device__ __forceinline__ float bilin_mix(const BilinAxis& y, const BilinAxis& x, float a, float b, float c, float d) {
  return y.h * (x.h * a + x.l * b) + y.l * (x.h * c + x.l * d);
}

// the value at output pixel (yo, xo) of an fp32 plane pl [H][W] up-sampled by f
__device__ __forceinline__ float bilin_at(const float* __restrict__ pl, int H, int W, int f, int yo, int xo) {
  const BilinAxis y = bilin_axis(yo, H, f), x = bilin_axis(xo, W, f);
  const float* r0 = pl + (size_t)y.i0 * W;
  const float* r1 = pl + (size_t)y.i1 * W;
  return bilin_mix(y, x, __ldg(r0 + x.i0), __ldg(r0 + x.i1), __ldg(r1 + x.i0), __ldg(r1 + x.i1));
}

// weight of source sample s in output coordinate o (n source samples, factor f), exactly as bilin_axis forms it: the
// coefficient the adjoint (a gather over each source sample's output footprint) multiplies that output by
__device__ __forceinline__ float bilin_tap(int o, int s, int n, int f) {
  const BilinAxis a = bilin_axis(o, n, f);
  return (a.i0 == s ? a.h : 0.f) + (a.i1 == s ? a.l : 0.f);
}

// (csrc/upsample2.cu) dx [N,h,w,C] = up2^T(dz) for fp32 NHWC dy [N,2h,2w,C], dz = dy where ymask > 0 and 0 elsewhere
// (ymask: the forward output of a ReLU epilogue, or NULL for dz = dy); C % 4 == 0, 16-byte aligned.  The GroupNorm
// backward's residual gradient in UPSNET_EPI_RES_BILINEAR mode, and upsnet_upsample2_bilinear_nhwc_adjoint.
int up2_bilinear_adjoint_launch(const float* dy, const float* ymask, float* dx, int N, int h, int w, int C,
                                cudaStream_t stream);

}  // namespace ups
