// roi_sample.cuh -- the ROIAlign sample rule, shared by every kernel that samples a map the way ROIAlign does
// (roi_align.cu's forward kernels, train_loss.cu's fused ROI loss and its backward gather).
//
// Semantics follow operators/src/roi_align_kernel.cu:43-95 (bilinear) and :163-235 (forward) of the reference: no
// half-pixel shift, roi extent forced >= 1, sampling grid gh x gw per bin, out-of-map test y<-1 || y>H.
#pragma once

namespace ups {

struct SamplePos {
  int o00, o01, o10, o11;  // element offsets (in pixels) of the four taps
  float w00, w01, w10, w11;
};

// the sample (y, x) lies inside the map's sampling range: ROIAlign gives an outside sample the value 0
__device__ __forceinline__ bool roi_sample_inside(int H, int W, float y, float x) {
  return !(y < -1.0f || y > (float)H || x < -1.0f || x > (float)W);
}

// roi_align_kernel.cu:43-95 -- returns weights/offsets instead of the value so that the NHWC
// kernel can reuse them across channels.  An out-of-range sample has all weights 0.
__device__ __forceinline__ SamplePos roi_sample(int H, int W, float y, float x) {
  SamplePos s;
  if (!roi_sample_inside(H, W, y, x)) {
    s.o00 = s.o01 = s.o10 = s.o11 = 0;
    s.w00 = s.w01 = s.w10 = s.w11 = 0.f;
    return s;
  }
  if (y <= 0) y = 0;
  if (x <= 0) x = 0;
  int yl = (int)y, xl = (int)x, yh, xh;
  if (yl >= H - 1) { yh = yl = H - 1; y = (float)yl; } else yh = yl + 1;
  if (xl >= W - 1) { xh = xl = W - 1; x = (float)xl; } else xh = xl + 1;
  const float ly = y - yl, lx = x - xl, hy = 1.f - ly, hx = 1.f - lx;
  s.o00 = yl * W + xl; s.o01 = yl * W + xh; s.o10 = yh * W + xl; s.o11 = yh * W + xh;
  s.w00 = hy * hx; s.w01 = hy * lx; s.w10 = ly * hx; s.w11 = ly * lx;
  return s;
}

// The bin geometry of one roi (x1, y1, x2, y2 in image coordinates) on a map at spatial scale sc, PH x PW bins.
struct RoiBins {
  float rsw, rsh;   // scaled start
  float bsw, bsh;   // bin size
};

__device__ __forceinline__ RoiBins roi_bins(float rx1, float ry1, float rx2, float ry2, float sc, int PH, int PW) {
  RoiBins b;
  b.rsw = rx1 * sc; b.rsh = ry1 * sc;
  const float rew = rx2 * sc, reh = ry2 * sc;
  const float rw = fmaxf(rew - b.rsw, 1.f), rh = fmaxf(reh - b.rsh, 1.f);
  b.bsh = rh / (float)PH; b.bsw = rw / (float)PW;
  return b;
}

// coordinate of sample i (0..g-1) of bin p along one axis: start + p * bin + (i + 0.5) * bin / g, with the roundings
// spelled out (p * bin + start fused), so that a caller whose i or g is a compile-time constant gets the same bits
__device__ __forceinline__ float roi_sample_coord(float start, int p, float bin, int i, int g) {
  return __fadd_rn(__fmaf_rn((float)p, bin, start), __fdiv_rn(__fmul_rn((float)(i + .5f), bin), (float)g));
}

}  // namespace ups
