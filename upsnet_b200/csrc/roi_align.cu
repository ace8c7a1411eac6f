// roi_align.cu -- ROIAlign / FPN-ROIAlign forward for sm_90a.
//
// Semantics follow operators/src/roi_align_kernel.cu:43-95 (bilinear) and :163-235 (forward)
// of the reference: no half-pixel shift, roi extent forced >= 1, sampling grid sr x sr,
// out-of-map test y<-1 || y>H.  The FPN variant folds fpn_roi_align.py:32-62 (level
// assignment, four per-level launches, cat + index_select) into one launch.
//
// Two data layouts:
//   NCHW  (reference API parity): thread per output element, pw fastest.
//   NHWC  (engine layout): one CTA per (roi, ph), lanes over channels -> every bilinear tap is
//         one contiguous C*4-byte read and every output write is coalesced.
// HBM-bound gather: algorithmic bytes = 4*R*C*PH*PW (write) + unique feature reads (DESIGN.md).
#include <cuda_bf16.h>

#include "common.cuh"
#include "pair.cuh"

namespace ups {

struct FpnFeats {
  const void* p[4];   // fp32, or bf16 for the NHWC engine layout
  int H[4], W[4];
  float scale[4];
  int nlevels;  // 1 => plain RoIAlign (level 0 always)
};

// Level thresholds on x = sqrtf(w*h)/224 + 1e-6 (float32): level = #{t : x >= thr[t]}.
// They are the smallest float32 x for which numpy's floor(2+log2(x)) reaches 1, 2, 3
// (fpn_roi_align.py:37 evaluated in float32): 0.5, 1.0 and 1.9999999 -- the last sits one ulp
// below 2 because 2 + log2f(x) rounds up to 3.0 there.  Pinned by tests/test_host_logic.py.
__device__ __forceinline__ int fpn_level_of(float x1, float y1, float x2, float y2) {
  const float w = x2 - x1 + 1.f, h = y2 - y1 + 1.f;
  const float x = __fadd_rn(__fdiv_rn(__fsqrt_rn(__fmul_rn(w, h)), 224.f), 1e-6f);
  const float t1 = __uint_as_float(0x3f000000u);  // 0.5
  const float t2 = __uint_as_float(0x3f800000u);  // 1.0
  const float t3 = __uint_as_float(0x3fffffffu);  // 1.9999999
  return (x >= t1) + (x >= t2) + (x >= t3);
}

struct SamplePos {
  int o00, o01, o10, o11;  // element offsets (in pixels) of the four taps
  float w00, w01, w10, w11;
};

// roi_align_kernel.cu:43-95 -- returns weights/offsets instead of the value so that the NHWC
// kernel can reuse them across channels.  An out-of-range sample has all weights 0.
__device__ __forceinline__ SamplePos roi_sample(int H, int W, float y, float x) {
  SamplePos s;
  if (y < -1.0f || y > (float)H || x < -1.0f || x > (float)W) {
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

// ------------------------------------------------------------------------------------------
// NCHW: thread per output element (n, c, ph, pw)
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
roi_align_nchw_kernel(FpnFeats f, int C, const float* __restrict__ rois, int R, int PH, int PW,
                      int sr, float* __restrict__ out, int* __restrict__ levels_out) {
  const long long total = (long long)R * C * PH * PW;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int pw = (int)(idx % PW);
    const int ph = (int)((idx / PW) % PH);
    const int c = (int)((idx / PW / PH) % C);
    const int n = (int)(idx / PW / PH / C);
    const float* r = rois + (size_t)n * 5;
    const int b = (int)roundf(r[0]);
    const float rx1 = r[1], ry1 = r[2], rx2 = r[3], ry2 = r[4];
    const int lv = f.nlevels > 1 ? fpn_level_of(rx1, ry1, rx2, ry2) : 0;
    if (levels_out && c == 0 && ph == 0 && pw == 0) levels_out[n] = lv;
    const int H = f.H[lv], W = f.W[lv];
    const float sc = f.scale[lv];
    const float rsw = rx1 * sc, rsh = ry1 * sc, rew = rx2 * sc, reh = ry2 * sc;
    const float rw = fmaxf(rew - rsw, 1.f), rh = fmaxf(reh - rsh, 1.f);
    const float bsh = rh / (float)PH, bsw = rw / (float)PW;
    const int gh = sr > 0 ? sr : (int)ceilf(rh / PH), gw = sr > 0 ? sr : (int)ceilf(rw / PW);
    const float* d = reinterpret_cast<const float*>(f.p[lv]) + ((size_t)b * C + c) * H * W;
    float acc = 0.f;
    for (int iy = 0; iy < gh; ++iy) {
      const float y = rsh + ph * bsh + (float)(iy + .5f) * bsh / (float)gh;
      for (int ix = 0; ix < gw; ++ix) {
        const float x = rsw + pw * bsw + (float)(ix + .5f) * bsw / (float)gw;
        const SamplePos s = roi_sample(H, W, y, x);
        acc += (s.w00 * __ldg(d + s.o00) + s.w01 * __ldg(d + s.o01) + s.w10 * __ldg(d + s.o10) +
                s.w11 * __ldg(d + s.o11));
      }
    }
    out[idx] = acc / (float)(gh * gw);
  }
}

// ------------------------------------------------------------------------------------------
// NHWC: CTA per (roi, ph); threads over channels (float4 per thread); loop over pw.
// ------------------------------------------------------------------------------------------
template <int VEC>
__global__ void __launch_bounds__(256)
roi_align_nhwc_kernel(FpnFeats f, int C, const float* __restrict__ rois, int R, int PH, int PW,
                      int sr, float* __restrict__ out, int* __restrict__ levels_out) {
  const int n = blockIdx.x / PH, ph = blockIdx.x % PH;
  const float* r = rois + (size_t)n * 5;
  const int b = (int)roundf(r[0]);
  const float rx1 = r[1], ry1 = r[2], rx2 = r[3], ry2 = r[4];
  const int lv = f.nlevels > 1 ? fpn_level_of(rx1, ry1, rx2, ry2) : 0;
  if (levels_out && ph == 0 && threadIdx.x == 0) levels_out[n] = lv;
  const int H = f.H[lv], W = f.W[lv];
  const float sc = f.scale[lv];
  const float rsw = rx1 * sc, rsh = ry1 * sc, rew = rx2 * sc, reh = ry2 * sc;
  const float rw = fmaxf(rew - rsw, 1.f), rh = fmaxf(reh - rsh, 1.f);
  const float bsh = rh / (float)PH, bsw = rw / (float)PW;
  const int gh = sr > 0 ? sr : (int)ceilf(rh / PH), gw = sr > 0 ? sr : (int)ceilf(rw / PW);
  const float inv_count_div = (float)(gh * gw);
  const float* base = reinterpret_cast<const float*>(f.p[lv]) + (size_t)b * H * W * C;
  for (int c = threadIdx.x * VEC; c < C; c += blockDim.x * VEC) {
    for (int pw = 0; pw < PW; ++pw) {
      float acc[VEC];
#pragma unroll
      for (int v = 0; v < VEC; ++v) acc[v] = 0.f;
      for (int iy = 0; iy < gh; ++iy) {
        const float y = rsh + ph * bsh + (float)(iy + .5f) * bsh / (float)gh;
        for (int ix = 0; ix < gw; ++ix) {
          const float x = rsw + pw * bsw + (float)(ix + .5f) * bsw / (float)gw;
          const SamplePos s = roi_sample(H, W, y, x);
          if (VEC == 4) {
            const float4 v00 = __ldg((const float4*)(base + (size_t)s.o00 * C + c));
            const float4 v01 = __ldg((const float4*)(base + (size_t)s.o01 * C + c));
            const float4 v10 = __ldg((const float4*)(base + (size_t)s.o10 * C + c));
            const float4 v11 = __ldg((const float4*)(base + (size_t)s.o11 * C + c));
            acc[0] += (s.w00 * v00.x + s.w01 * v01.x + s.w10 * v10.x + s.w11 * v11.x);
            acc[1 % VEC] += (s.w00 * v00.y + s.w01 * v01.y + s.w10 * v10.y + s.w11 * v11.y);
            acc[2 % VEC] += (s.w00 * v00.z + s.w01 * v01.z + s.w10 * v10.z + s.w11 * v11.z);
            acc[3 % VEC] += (s.w00 * v00.w + s.w01 * v01.w + s.w10 * v10.w + s.w11 * v11.w);
          } else {
            acc[0] += (s.w00 * __ldg(base + (size_t)s.o00 * C + c) +
                       s.w01 * __ldg(base + (size_t)s.o01 * C + c) +
                       s.w10 * __ldg(base + (size_t)s.o10 * C + c) +
                       s.w11 * __ldg(base + (size_t)s.o11 * C + c));
          }
        }
      }
      float* o = out + (((size_t)n * PH + ph) * PW + pw) * C + c;
      if (VEC == 4) {
        float4 v;
        v.x = acc[0] / inv_count_div; v.y = acc[1 % VEC] / inv_count_div;
        v.z = acc[2 % VEC] / inv_count_div; v.w = acc[3 % VEC] / inv_count_div;
        *(float4*)o = v;
      } else {
        o[0] = acc[0] / inv_count_div;
      }
    }
  }
}

// NHWC, bf16 features in / bf16 out (engine layout when activations are stored as bf16): lanes over channel
// quads (8-byte loads), fp32 accumulation, same sample arithmetic.
__global__ void __launch_bounds__(256)
roi_align_nhwc_bf16_kernel(FpnFeats f, int C, const float* __restrict__ rois, int R, int PH, int PW, int sr,
                           __nv_bfloat16* __restrict__ out, int* __restrict__ levels_out) {
  const int n = blockIdx.x / PH, ph = blockIdx.x % PH;
  const float* r = rois + (size_t)n * 5;
  const int b = (int)roundf(r[0]);
  const float rx1 = r[1], ry1 = r[2], rx2 = r[3], ry2 = r[4];
  const int lv = f.nlevels > 1 ? fpn_level_of(rx1, ry1, rx2, ry2) : 0;
  if (levels_out && ph == 0 && threadIdx.x == 0) levels_out[n] = lv;
  const int H = f.H[lv], W = f.W[lv];
  const float sc = f.scale[lv];
  const float rsw = rx1 * sc, rsh = ry1 * sc, rew = rx2 * sc, reh = ry2 * sc;
  const float rw = fmaxf(rew - rsw, 1.f), rh = fmaxf(reh - rsh, 1.f);
  const float bsh = rh / (float)PH, bsw = rw / (float)PW;
  const int gh = sr > 0 ? sr : (int)ceilf(rh / PH), gw = sr > 0 ? sr : (int)ceilf(rw / PW);
  const float cnt = (float)(gh * gw);
  const __nv_bfloat16* base = reinterpret_cast<const __nv_bfloat16*>(f.p[lv]) + (size_t)b * H * W * C;
  for (int c = threadIdx.x * 4; c < C; c += blockDim.x * 4) {
    for (int pw = 0; pw < PW; ++pw) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int iy = 0; iy < gh; ++iy) {
        const float y = rsh + ph * bsh + (float)(iy + .5f) * bsh / (float)gh;
        for (int ix = 0; ix < gw; ++ix) {
          const float x = rsw + pw * bsw + (float)(ix + .5f) * bsw / (float)gw;
          const SamplePos s = roi_sample(H, W, y, x);
          const uint2 v00 = __ldg(reinterpret_cast<const uint2*>(base + (size_t)s.o00 * C + c));
          const uint2 v01 = __ldg(reinterpret_cast<const uint2*>(base + (size_t)s.o01 * C + c));
          const uint2 v10 = __ldg(reinterpret_cast<const uint2*>(base + (size_t)s.o10 * C + c));
          const uint2 v11 = __ldg(reinterpret_cast<const uint2*>(base + (size_t)s.o11 * C + c));
          const uint32_t a[2] = {v00.x, v00.y}, bq[2] = {v01.x, v01.y}, d[2] = {v10.x, v10.y}, e[2] = {v11.x, v11.y};
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            acc[2 * q] += (s.w00 * bf16x2_x(a[q]) + s.w01 * bf16x2_x(bq[q]) + s.w10 * bf16x2_x(d[q]) + s.w11 * bf16x2_x(e[q]));
            acc[2 * q + 1] += (s.w00 * bf16x2_y(a[q]) + s.w01 * bf16x2_y(bq[q]) + s.w10 * bf16x2_y(d[q]) + s.w11 * bf16x2_y(e[q]));
          }
        }
      }
      const uint2 w = make_uint2(pack_bf16x2(acc[0] / cnt, acc[1] / cnt), pack_bf16x2(acc[2] / cnt, acc[3] / cnt));
      *reinterpret_cast<uint2*>(out + (((size_t)n * PH + ph) * PW + pw) * C + c) = w;
    }
  }
}

// Same operator, CTA = one roi: the PH*PW*gh*gw sample positions (offsets + bilinear weights) are computed ONCE
// into shared memory, then every warp takes bins round-robin with lanes over 8-channel (16-byte) vectors -- the
// per-sample arithmetic is no longer repeated by every channel quad, and loads are twice as wide.  Accumulation
// order (iy, ix; four-term blend) is the one of the kernel above, so results are bit-identical.
constexpr int kRoiMaxSamples = 1024;
__global__ void __launch_bounds__(256)
roi_align_nhwc_bf16_roi_kernel(FpnFeats f, int C, const float* __restrict__ rois, int R, int PH, int PW, int sr,
                               __nv_bfloat16* __restrict__ out, int* __restrict__ levels_out) {
  __shared__ int4 s_off[kRoiMaxSamples];
  __shared__ float4 s_w[kRoiMaxSamples];
  const int n = blockIdx.x;
  const float* r = rois + (size_t)n * 5;
  const int b = (int)roundf(r[0]);
  const float rx1 = r[1], ry1 = r[2], rx2 = r[3], ry2 = r[4];
  const int lv = f.nlevels > 1 ? fpn_level_of(rx1, ry1, rx2, ry2) : 0;
  if (levels_out && threadIdx.x == 0) levels_out[n] = lv;
  const int H = f.H[lv], W = f.W[lv];
  const float sc = f.scale[lv];
  const float rsw = rx1 * sc, rsh = ry1 * sc, rew = rx2 * sc, reh = ry2 * sc;
  const float rw = fmaxf(rew - rsw, 1.f), rh = fmaxf(reh - rsh, 1.f);
  const float bsh = rh / (float)PH, bsw = rw / (float)PW;
  const int gh = sr, gw = sr;                 // launcher guarantees sr > 0 and PH*PW*sr*sr <= kRoiMaxSamples
  const float cnt = (float)(gh * gw);
  const int per_bin = gh * gw, nsamp = PH * PW * per_bin;
  for (int t = threadIdx.x; t < nsamp; t += blockDim.x) {
    const int bin = t / per_bin, q = t - bin * per_bin;
    const int ph = bin / PW, pw = bin - ph * PW, iy = q / gw, ix = q - iy * gw;
    const float y = rsh + ph * bsh + (float)(iy + .5f) * bsh / (float)gh;
    const float x = rsw + pw * bsw + (float)(ix + .5f) * bsw / (float)gw;
    const SamplePos sp = roi_sample(H, W, y, x);
    s_off[t] = make_int4(sp.o00 * C, sp.o01 * C, sp.o10 * C, sp.o11 * C);
    s_w[t] = make_float4(sp.w00, sp.w01, sp.w10, sp.w11);
  }
  __syncthreads();
  const __nv_bfloat16* base = reinterpret_cast<const __nv_bfloat16*>(f.p[lv]) + (size_t)b * H * W * C;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
  for (int bin = warp; bin < PH * PW; bin += nwarp) {
    for (int c = lane * 8; c < C; c += 256) {
      float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int q = 0; q < per_bin; ++q) {
        const int4 o = s_off[bin * per_bin + q];
        const float4 w = s_w[bin * per_bin + q];
        const uint4 v00 = __ldg(reinterpret_cast<const uint4*>(base + o.x + c));
        const uint4 v01 = __ldg(reinterpret_cast<const uint4*>(base + o.y + c));
        const uint4 v10 = __ldg(reinterpret_cast<const uint4*>(base + o.z + c));
        const uint4 v11 = __ldg(reinterpret_cast<const uint4*>(base + o.w + c));
        const uint32_t a[4] = {v00.x, v00.y, v00.z, v00.w}, bq[4] = {v01.x, v01.y, v01.z, v01.w};
        const uint32_t d[4] = {v10.x, v10.y, v10.z, v10.w}, e[4] = {v11.x, v11.y, v11.z, v11.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          acc[2 * k] += (w.x * bf16x2_x(a[k]) + w.y * bf16x2_x(bq[k]) + w.z * bf16x2_x(d[k]) + w.w * bf16x2_x(e[k]));
          acc[2 * k + 1] += (w.x * bf16x2_y(a[k]) + w.y * bf16x2_y(bq[k]) + w.z * bf16x2_y(d[k]) + w.w * bf16x2_y(e[k]));
        }
      }
      const uint4 wv = make_uint4(pack_bf16x2(acc[0] / cnt, acc[1] / cnt), pack_bf16x2(acc[2] / cnt, acc[3] / cnt),
                                  pack_bf16x2(acc[4] / cnt, acc[5] / cnt), pack_bf16x2(acc[6] / cnt, acc[7] / cnt));
      *reinterpret_cast<uint4*>(out + ((size_t)n * PH * PW + bin) * C + c) = wv;
    }
  }
}

// hi/lo pair features in ([B,H,W,2C] bf16 per level), pair result out: the blend runs on hi + lo (exact in fp32) and the
// fp32 bin average is split again.  Output addressing is (roi_stride, pix_stride, lo_off) in elements:
//   pair pixels [R,PH,PW,2C]   (mask branch: the 14x14 roi maps feed 3x3 convs)   -> (PH*PW*2C, 2C, C)
//   flat pair   [R,2,PH*PW*C]  (RCNN fc6: one 'pixel' per roi with PH*PW*C channels) -> (2*PH*PW*C, C, PH*PW*C)
// Same sample arithmetic and accumulation order as the bf16 / fp32 kernels above.
__global__ void __launch_bounds__(256)
roi_align_nhwc_pair_roi_kernel(FpnFeats f, int C, const float* __restrict__ rois, int R, int PH, int PW, int sr,
                               __nv_bfloat16* __restrict__ out, long long roi_stride, int pix_stride, long long lo_off,
                               int* __restrict__ levels_out, const int* __restrict__ n_dev) {
  __shared__ int4 s_off[kRoiMaxSamples];
  __shared__ float4 s_w[kRoiMaxSamples];
  const int n = blockIdx.x;
  if (n_dev && n >= *n_dev) return;     // rois beyond the device-side count: neither read nor written
  const float* r = rois + (size_t)n * 5;
  const int b = (int)roundf(r[0]);
  const float rx1 = r[1], ry1 = r[2], rx2 = r[3], ry2 = r[4];
  const int lv = f.nlevels > 1 ? fpn_level_of(rx1, ry1, rx2, ry2) : 0;
  if (levels_out && threadIdx.x == 0) levels_out[n] = lv;
  const int H = f.H[lv], W = f.W[lv];
  const float sc = f.scale[lv];
  const float rsw = rx1 * sc, rsh = ry1 * sc, rew = rx2 * sc, reh = ry2 * sc;
  const float rw = fmaxf(rew - rsw, 1.f), rh = fmaxf(reh - rsh, 1.f);
  const float bsh = rh / (float)PH, bsw = rw / (float)PW;
  const int gh = sr, gw = sr;
  const float cnt = (float)(gh * gw);
  const int per_bin = gh * gw, nsamp = PH * PW * per_bin;
  for (int t = threadIdx.x; t < nsamp; t += blockDim.x) {
    const int bin = t / per_bin, q = t - bin * per_bin;
    const int ph = bin / PW, pw = bin - ph * PW, iy = q / gw, ix = q - iy * gw;
    const float y = rsh + ph * bsh + (float)(iy + .5f) * bsh / (float)gh;
    const float x = rsw + pw * bsw + (float)(ix + .5f) * bsw / (float)gw;
    const SamplePos sp = roi_sample(H, W, y, x);
    s_off[t] = make_int4(sp.o00 * 2 * C, sp.o01 * 2 * C, sp.o10 * 2 * C, sp.o11 * 2 * C);
    s_w[t] = make_float4(sp.w00, sp.w01, sp.w10, sp.w11);
  }
  __syncthreads();
  const __nv_bfloat16* base = reinterpret_cast<const __nv_bfloat16*>(f.p[lv]) + (size_t)b * H * W * 2 * C;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
  for (int bin = warp; bin < PH * PW; bin += nwarp) {
    for (int c = lane * 8; c < C; c += 256) {
      float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int q = 0; q < per_bin; ++q) {
        const int4 o = s_off[bin * per_bin + q];
        const float4 w = s_w[bin * per_bin + q];
        const __nv_bfloat16* p0 = base + o.x + c; const __nv_bfloat16* p1 = base + o.y + c;
        const __nv_bfloat16* p2 = base + o.z + c; const __nv_bfloat16* p3 = base + o.w + c;
        const uint4 h0 = __ldg(reinterpret_cast<const uint4*>(p0)), l0 = __ldg(reinterpret_cast<const uint4*>(p0 + C));
        const uint4 h1 = __ldg(reinterpret_cast<const uint4*>(p1)), l1 = __ldg(reinterpret_cast<const uint4*>(p1 + C));
        const uint4 h2 = __ldg(reinterpret_cast<const uint4*>(p2)), l2 = __ldg(reinterpret_cast<const uint4*>(p2 + C));
        const uint4 h3 = __ldg(reinterpret_cast<const uint4*>(p3)), l3 = __ldg(reinterpret_cast<const uint4*>(p3 + C));
        const uint32_t A[4] = {h0.x, h0.y, h0.z, h0.w}, a[4] = {l0.x, l0.y, l0.z, l0.w};
        const uint32_t B[4] = {h1.x, h1.y, h1.z, h1.w}, bq[4] = {l1.x, l1.y, l1.z, l1.w};
        const uint32_t D[4] = {h2.x, h2.y, h2.z, h2.w}, d[4] = {l2.x, l2.y, l2.z, l2.w};
        const uint32_t E[4] = {h3.x, h3.y, h3.z, h3.w}, e[4] = {l3.x, l3.y, l3.z, l3.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          acc[2 * k] += (w.x * pair_x(A[k], a[k]) + w.y * pair_x(B[k], bq[k]) + w.z * pair_x(D[k], d[k]) + w.w * pair_x(E[k], e[k]));
          acc[2 * k + 1] += (w.x * pair_y(A[k], a[k]) + w.y * pair_y(B[k], bq[k]) + w.z * pair_y(D[k], d[k]) + w.w * pair_y(E[k], e[k]));
        }
      }
      uint32_t hw[4], lw[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) split_pair2(acc[2 * k] / cnt, acc[2 * k + 1] / cnt, hw[k], lw[k]);
      __nv_bfloat16* op = out + (size_t)n * roi_stride + (size_t)bin * pix_stride + c;
      *reinterpret_cast<uint4*>(op) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
      *reinterpret_cast<uint4*>(op + lo_off) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
    }
  }
}

static int launch_roi_align(const FpnFeats& f, int B, int C, int layout, int dtype, const float* rois, int R,
                            int PH, int PW, int sr, void* out_v, int* levels_out, const int* n_dev,
                            cudaStream_t stream) {
  if (R < 0 || C <= 0 || PH <= 0 || PW <= 0 || B <= 0) return UPSNET_E_BADARG;
  if (R == 0) return 0;
  if (n_dev && dtype != UPSNET_DTYPE_PAIR) return UPSNET_E_UNSUPPORTED;
  if (dtype == UPSNET_DTYPE_PAIR) {
    if (layout != UPSNET_LAYOUT_NHWC && layout != UPSNET_LAYOUT_FLAT_PAIR) return UPSNET_E_UNSUPPORTED;
    if (sr <= 0 || (C & 7) || (long long)PH * PW * sr * sr > kRoiMaxSamples || (((uintptr_t)out_v) & 15)) return UPSNET_E_UNSUPPORTED;
    for (int l = 0; l < f.nlevels; ++l)
      if ((((uintptr_t)f.p[l]) & 15) || (long long)f.H[l] * f.W[l] * 2 * C >= (1ll << 31)) return UPSNET_E_UNSUPPORTED;
    const long long plane = (long long)PH * PW * C;
    const bool flat = layout == UPSNET_LAYOUT_FLAT_PAIR;
    roi_align_nhwc_pair_roi_kernel<<<R, 256, 0, stream>>>(f, C, rois, R, PH, PW, sr, (__nv_bfloat16*)out_v, 2 * plane,
                                                          flat ? C : 2 * C, flat ? plane : (long long)C, levels_out, n_dev);
    UPS_CHECK_LAUNCH();
    return 0;
  }
  if (dtype == UPSNET_DTYPE_BF16) {
    if (layout != UPSNET_LAYOUT_NHWC || (C & 3)) return UPSNET_E_UNSUPPORTED;
    for (int l = 0; l < f.nlevels; ++l) if (((uintptr_t)f.p[l]) & 7) return UPSNET_E_BADARG;
    if (((uintptr_t)out_v) & 7) return UPSNET_E_BADARG;
    bool wide = sr > 0 && (C & 7) == 0 && (long long)PH * PW * sr * sr <= kRoiMaxSamples && (((uintptr_t)out_v) & 15) == 0;
    for (int l = 0; l < f.nlevels; ++l) wide = wide && (((uintptr_t)f.p[l]) & 15) == 0 && (long long)f.H[l] * f.W[l] * C < (1ll << 31);
    if (wide) {
      roi_align_nhwc_bf16_roi_kernel<<<R, 256, 0, stream>>>(f, C, rois, R, PH, PW, sr, (__nv_bfloat16*)out_v, levels_out);
      UPS_CHECK_LAUNCH();
      return 0;
    }
    const int threads = C / 4 < 32 ? 32 : (C / 4 > 256 ? 256 : (C / 4 + 31) / 32 * 32);
    roi_align_nhwc_bf16_kernel<<<R * PH, threads, 0, stream>>>(f, C, rois, R, PH, PW, sr, (__nv_bfloat16*)out_v, levels_out);
    UPS_CHECK_LAUNCH();
    return 0;
  }
  if (dtype != UPSNET_DTYPE_F32) return UPSNET_E_BADARG;
  float* out = reinterpret_cast<float*>(out_v);
  if (layout == UPSNET_LAYOUT_NCHW) {
    const long long total = (long long)R * C * PH * PW;
    long long blocks = (total + 255) / 256;
    if (blocks > kNumSMs * 64) blocks = kNumSMs * 64;
    roi_align_nchw_kernel<<<(int)blocks, 256, 0, stream>>>(f, C, rois, R, PH, PW, sr, out,
                                                           levels_out);
  } else if (layout == UPSNET_LAYOUT_NHWC) {
    bool vec4 = (C % 4 == 0);
    for (int l = 0; l < f.nlevels; ++l) vec4 = vec4 && (((uintptr_t)f.p[l] & 15) == 0);
    vec4 = vec4 && (((uintptr_t)out & 15) == 0);
    if (vec4) {
      int threads = C / 4 < 32 ? 32 : (C / 4 > 256 ? 256 : (C / 4 + 31) / 32 * 32);
      roi_align_nhwc_kernel<4><<<R * PH, threads, 0, stream>>>(f, C, rois, R, PH, PW, sr, out,
                                                              levels_out);
    } else {
      int threads = C < 32 ? 32 : (C > 256 ? 256 : (C + 31) / 32 * 32);
      roi_align_nhwc_kernel<1><<<R * PH, threads, 0, stream>>>(f, C, rois, R, PH, PW, sr, out,
                                                              levels_out);
    }
  } else {
    return UPSNET_E_BADARG;
  }
  UPS_CHECK_LAUNCH();
  return 0;
}

}  // namespace ups

extern "C" int upsnet_roi_align_forward(const void* feat, int B, int C, int H, int W, int layout, int dtype,
                                        const float* rois, int R, int PH, int PW,
                                        int sampling_ratio, float spatial_scale, void* out,
                                        void* stream) {
  if (!feat || !out || (!rois && R > 0)) return UPSNET_E_BADARG;
  ups::FpnFeats f{};
  f.p[0] = feat; f.H[0] = H; f.W[0] = W; f.scale[0] = spatial_scale; f.nlevels = 1;
  return ups::launch_roi_align(f, B, C, layout, dtype, rois, R, PH, PW, sampling_ratio, out, nullptr, nullptr,
                               (cudaStream_t)stream);
}

extern "C" int upsnet_roi_align_fpn_forward(const void* const feats[4], const int Hs[4],
                                            const int Ws[4], const float scales[4], int B, int C,
                                            int layout, int dtype, const float* rois, int R, int PH, int PW,
                                            int sampling_ratio, void* out, int* levels_out,
                                            const int* n_dev, void* stream) {
  if (!feats || !Hs || !Ws || !scales || !out || (!rois && R > 0)) return UPSNET_E_BADARG;
  ups::FpnFeats f{};
  for (int l = 0; l < 4; ++l) {
    if (!feats[l]) return UPSNET_E_BADARG;
    f.p[l] = feats[l]; f.H[l] = Hs[l]; f.W[l] = Ws[l]; f.scale[l] = scales[l];
  }
  f.nlevels = 4;
  return ups::launch_roi_align(f, B, C, layout, dtype, rois, R, PH, PW, sampling_ratio, out, levels_out, n_dev,
                               (cudaStream_t)stream);
}
