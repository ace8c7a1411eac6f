// post.cu -- the two callers either side of the per-image forward (SURVEY section 8f rows f2, f3), device resident:
//
//  * upsnet_unified_pan_result: dataset/base_dataset.py:332-371 get_unified_pan_result -- per-instance majority vote of
//    the semantic labels under every panoptic instance segment, the stuff-area limit, and the 2-channel (class, instance)
//    map the PQ evaluation consumes.  Reference: numpy on the host after two [H,W] D2H copies, np.unique per segment.
//    Here: one warp-aggregated histogram pass, one tiny decision kernel, one relabel pass, one area-limit pass.
//  * upsnet_prep_image: dataset/base_dataset.py:143-174 prep_im_for_blob + :898-923 im_list_to_blob -- mean subtraction,
//    bilinear resize (cv2.INTER_LINEAR rule) and zero padding to a multiple of the FPN stride, uint8 HWC BGR in, fp32 NCHW
//    out.  Reference: numpy + cv2 on the host, then a 4x larger fp32 H2D copy.
//  * upsnet_label_restore: upsnet_end2end_test.py:259-266 (row f4) -- both label maps cropped to im_info[:2], wrapped to
//    uint8 and resized back to the original image size with cv2's INTER_NEAREST rule, in one launch.
// All are HBM-bound streaming kernels (bytes: 16*H*W + 3*H*W; 3*h*w + 12*Hp*Wp; 16*oh*ow per map).
#include "common.cuh"

namespace ups {

constexpr int kUniMaxInst = 256;   // instance ids are < 255 (255 = void): at most 254 - id_last_stuff instances
constexpr int kUniMaxCls = 256;

struct UniWs {
  int* hist;             // [kUniMaxInst][S]
  int* present;          // [kUniMaxInst]
  int* area;             // [kUniMaxCls]
  int* err;              // [1]
  unsigned char* seg_of; // [kUniMaxInst]
  unsigned char* ins_of; // [kUniMaxInst]
};

static size_t uni_ws_layout(int S, UniWs& ws, void* base) {
  WsCarve c(base);
  ws.hist = c.take<int>((size_t)kUniMaxInst * S);
  ws.present = c.take<int>(kUniMaxInst);
  ws.area = c.take<int>(kUniMaxCls);
  ws.err = c.take<int>(1);
  ws.seg_of = c.take<unsigned char>(kUniMaxInst);
  ws.ins_of = c.take<unsigned char>(kUniMaxInst);
  return c.bytes();
}

// (instance, semantic class) histogram.  Neighbouring pixels mostly share both keys, so the lanes of a warp that hold the
// same key elect one leader that adds their count (warp-aggregated atomics): ~1 atomic per warp instead of 32.
__global__ void __launch_bounds__(256)
uni_hist_kernel(const long long* __restrict__ seg, const long long* __restrict__ pan, size_t HW, int id_last, int S, UniWs ws) {
  for (size_t p0 = (size_t)blockIdx.x * blockDim.x; p0 < HW; p0 += (size_t)gridDim.x * blockDim.x) {
    const size_t p = p0 + threadIdx.x;
    int key = -1;
    if (p < HW) {
      const long long v = pan[p];
      if (v > id_last && v != 255) {
        const long long s = seg[p];
        if (v - id_last - 1 < kUniMaxInst && s >= 0 && s < S) key = (int)(v - id_last - 1) * S + (int)s;
        else atomicOr(ws.err, 1);
      }
    }
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    if (key >= 0 && (int)(__ffs(peers) - 1) == (int)(threadIdx.x & 31)) {
      atomicAdd(ws.hist + key, __popc(peers));
      ws.present[key / S] = 1;
    }
  }
}

// One thread per instance slot: majority class (first maximum = smallest class id, like np.unique + np.argmax), the rank
// among the PRESENT instance ids (pan_ins = rank + 1), and the three-way decision of base_dataset.py:349-358.
__global__ void __launch_bounds__(kUniMaxInst)
uni_decide_kernel(const long long* __restrict__ cls_ind, int k, const int* __restrict__ k_dev, int id_last, int S, UniWs ws) {
  __shared__ int s_pres[kUniMaxInst];
  const int j = threadIdx.x;
  const int kk = k_dev ? min(*k_dev, k) : k;
  s_pres[j] = ws.present[j];
  if (j < kUniMaxCls) ws.area[j] = 0;
  __syncthreads();
  if (!s_pres[j]) return;
  int rank = 0;
  for (int q = 0; q < j; ++q) rank += s_pres[q];
  if (j >= kk) { atomicOr(ws.err, 2); return; }       // a label without an entry in cls_inds: the reference raises IndexError
  long long total = 0;
  int best = 0, best_c = 0;
  for (int c = 0; c < S; ++c) {
    const int n = ws.hist[j * S + c];
    total += n;
    if (n > best) { best = n; best_c = c; }
  }
  const int target = (int)cls_ind[j] + id_last;
  int seg_v, ins_v;
  if (best_c == target) { seg_v = target; ins_v = rank + 1; }
  else if (2ll * best >= total && best_c <= id_last) { seg_v = best_c; ins_v = 0; }     // np.max(cnt) / np.sum(cnt) >= 0.5
  else { seg_v = target; ins_v = rank + 1; }
  ws.seg_of[j] = (unsigned char)seg_v;
  ws.ins_of[j] = (unsigned char)ins_v;
}

__global__ void __launch_bounds__(256)
uni_relabel_kernel(const long long* __restrict__ pan, size_t HW, int id_last, UniWs ws, unsigned char* __restrict__ out) {
  __shared__ int s_area[kUniMaxCls];
  for (int t = threadIdx.x; t < kUniMaxCls; t += blockDim.x) s_area[t] = 0;
  __syncthreads();
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (size_t)gridDim.x * blockDim.x) {
    const long long v = pan[p];
    int ps, pi = 0;
    if (v <= id_last) ps = (int)v;
    else if (v == 255 || v - id_last - 1 >= kUniMaxInst) ps = 255;
    else { ps = ws.seg_of[v - id_last - 1]; pi = ws.ins_of[v - id_last - 1]; }
    out[p * 3] = (unsigned char)ps; out[p * 3 + 1] = (unsigned char)pi; out[p * 3 + 2] = 0;
    if (ps >= 0 && ps <= id_last) atomicAdd(s_area + ps, 1);
  }
  __syncthreads();
  for (int t = threadIdx.x; t <= id_last && t < kUniMaxCls; t += blockDim.x)
    if (s_area[t]) atomicAdd(ws.area + t, s_area[t]);
}

__global__ void __launch_bounds__(256)
uni_area_kernel(size_t HW, int id_last, int stuff_area_limit, UniWs ws, unsigned char* __restrict__ out) {
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += (size_t)gridDim.x * blockDim.x) {
    const int ps = out[p * 3];
    if (ps <= id_last && ws.area[ps] < stuff_area_limit) out[p * 3] = 255;
  }
}

// ---- input pipeline ----
// cv2.resize INTER_LINEAR source coordinate (imgproc/resize.cpp): fx = (float)((dx + 0.5) * scale - 0.5) with the double
// scale = src / dst, floor, clamp at both borders with weight 0 -- the rule of oracle_mask_resize (oracle/upsnet_oracle.c).
__device__ __forceinline__ void lin_coef(int d, int n_src, double scale, int& s, float& f) {
  float fv = (float)__dadd_rn(__dmul_rn((double)d + 0.5, scale), -0.5);
  int sv = (int)floorf(fv);
  fv = __fsub_rn(fv, (float)sv);
  if (sv < 0) { sv = 0; fv = 0.f; }
  if (sv >= n_src - 1) { sv = n_src - 1; fv = 0.f; }
  s = sv; f = fv;
}

__global__ void __launch_bounds__(256)
prep_image_kernel(const unsigned char* __restrict__ src, int h, int w, int ho, int wo, int Hp, int Wp, double inv_scale,
                  double m0, double m1, double m2, int flip, float* __restrict__ out) {
  const size_t plane = (size_t)Hp * Wp;
  // cv2.resize(im, None, None, fx, fy): the source step is 1 / fx -- the given factor, NOT the ratio of the rounded sizes
  const double sx = inv_scale, sy = inv_scale;
  const bool same = (h == ho && w == wo);
  // flip: column x of the flipped image (get_image_blob's im[:, ::-1, :]) is source column w - 1 - x.  Every column index
  // goes through it after the tap geometry, so the result is the kernel's output for a host-flipped copy, bit for bit.
  const int xr = flip ? w - 1 : 0, xs = flip ? -1 : 1;
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < plane; p += (size_t)gridDim.x * blockDim.x) {
    const int y = (int)(p / Wp), x = (int)(p - (size_t)y * Wp);
    float v0 = 0.f, v1 = 0.f, v2 = 0.f;
    if (y < ho && x < wo) {
      if (same) {
        const unsigned char* q = src + ((size_t)y * w + (xr + xs * x)) * 3;
        v0 = (float)((double)q[0] - m0); v1 = (float)((double)q[1] - m1); v2 = (float)((double)q[2] - m2);   // numpy: float64 subtract, float32 store
      } else {
        int x0, y0; float fx, fy;
        lin_coef(x, w, sx, x0, fx);
        lin_coef(y, h, sy, y0, fy);
        const int x1 = xr + xs * min(x0 + 1, w - 1), y1 = min(y0 + 1, h - 1);
        x0 = xr + xs * x0;
        const unsigned char* a = src + ((size_t)y0 * w + x0) * 3; const unsigned char* b = src + ((size_t)y0 * w + x1) * 3;
        const unsigned char* c = src + ((size_t)y1 * w + x0) * 3; const unsigned char* d = src + ((size_t)y1 * w + x1) * 3;
        const float gx = __fsub_rn(1.f, fx), gy = __fsub_rn(1.f, fy);
        const double mean[3] = {m0, m1, m2};
        float r[3];
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {     // mean first (prep_im_for_blob:154), then rows, then columns, un-fused fp32
          const float A = (float)((double)a[ch] - mean[ch]), B = (float)((double)b[ch] - mean[ch]);
          const float C = (float)((double)c[ch] - mean[ch]), D = (float)((double)d[ch] - mean[ch]);
          const float top = __fadd_rn(__fmul_rn(A, gx), __fmul_rn(B, fx));
          const float bot = __fadd_rn(__fmul_rn(C, gx), __fmul_rn(D, fx));
          r[ch] = __fadd_rn(__fmul_rn(top, gy), __fmul_rn(bot, fy));
        }
        v0 = r[0]; v1 = r[1]; v2 = r[2];
      }
    }
    out[p] = v0; out[plane + p] = v1; out[2 * plane + p] = v2;
  }
}

// ---- label maps back to the original image size (upsnet_end2end_test.py:259-266) ----
// cv2.resize INTER_NEAREST (imgproc/resize.cpp resizeNN): ifx = 1 / fx in double, sx = min(cvFloor(x * ifx), w - 1).
// blockIdx.y picks the map; the crop [:h,:w] is the clamp, astype(uint8) the & 0xff.
__global__ void __launch_bounds__(256)
label_restore_kernel(const long long* __restrict__ src0, const long long* __restrict__ src1, int Wp, int h, int w,
                     double ifx, int out_h, int out_w, long long* __restrict__ dst0, long long* __restrict__ dst1) {
  const long long* src = blockIdx.y ? src1 : src0;
  long long* dst = blockIdx.y ? dst1 : dst0;
  const size_t n = (size_t)out_h * out_w;
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (size_t)gridDim.x * blockDim.x) {
    const int y = (int)(p / out_w), x = (int)(p - (size_t)y * out_w);
    const int sy = min((int)floor(__dmul_rn((double)y, ifx)), h - 1);
    const int sx = min((int)floor(__dmul_rn((double)x, ifx)), w - 1);
    dst[p] = (long long)(unsigned char)src[(size_t)sy * Wp + sx];
  }
}

}  // namespace ups

extern "C" int upsnet_unified_pan_workspace_bytes(int num_seg_classes, size_t* bytes) {
  if (!bytes || num_seg_classes <= 0 || num_seg_classes > ups::kUniMaxCls) return UPSNET_E_BADARG;
  ups::UniWs ws;
  *bytes = ups::uni_ws_layout(num_seg_classes, ws, nullptr);
  return 0;
}

extern "C" int upsnet_unified_pan_result(const long long* seg, const long long* pan, const long long* cls_inds, int k,
                                         const int* k_dev, int H, int W, int num_seg_classes, int num_classes,
                                         int stuff_area_limit, unsigned char* pan_2ch, int* err_out, void* workspace,
                                         size_t workspace_bytes, void* stream) {
  using namespace ups;
  if (!seg || !pan || !pan_2ch || !workspace || (!cls_inds && k > 0)) return UPSNET_E_BADARG;
  if (H <= 0 || W <= 0 || k < 0 || num_classes < 1 || num_seg_classes < num_classes || num_seg_classes > kUniMaxCls)
    return UPSNET_E_BADARG;
  UniWs ws;
  const size_t need = uni_ws_layout(num_seg_classes, ws, workspace);
  if (workspace_bytes < need) return UPSNET_E_WORKSPACE;
  const int id_last = num_seg_classes - num_classes;
  const size_t HW = (size_t)H * W;
  cudaStream_t st = (cudaStream_t)stream;
  UPS_CUDA(cudaMemsetAsync(workspace, 0, need, st));
  size_t blocks = (HW + 255) / 256;
  if (blocks > (size_t)kNumSMs * 16) blocks = (size_t)kNumSMs * 16;
  uni_hist_kernel<<<(unsigned)blocks, 256, 0, st>>>(seg, pan, HW, id_last, num_seg_classes, ws);
  UPS_CHECK_LAUNCH();
  uni_decide_kernel<<<1, kUniMaxInst, 0, st>>>(cls_inds, k, k_dev, id_last, num_seg_classes, ws);
  UPS_CHECK_LAUNCH();
  uni_relabel_kernel<<<(unsigned)blocks, 256, 0, st>>>(pan, HW, id_last, ws, pan_2ch);
  UPS_CHECK_LAUNCH();
  uni_area_kernel<<<(unsigned)blocks, 256, 0, st>>>(HW, id_last, stuff_area_limit, ws, pan_2ch);
  UPS_CHECK_LAUNCH();
  if (err_out) UPS_CUDA(cudaMemcpyAsync(err_out, ws.err, sizeof(int), cudaMemcpyDeviceToDevice, st));
  return 0;
}

extern "C" int upsnet_prep_image(const unsigned char* image_hwc, int h, int w, double scale, int out_h, int out_w, int pad_h,
                                 int pad_w, const double pixel_means[3], float* blob, int flip, void* stream) {
  if (!image_hwc || !blob || !pixel_means) return UPSNET_E_BADARG;
  if (h <= 0 || w <= 0 || out_h <= 0 || out_w <= 0 || pad_h < out_h || pad_w < out_w || !(scale > 0.0)) return UPSNET_E_BADARG;
  const size_t plane = (size_t)pad_h * pad_w;
  size_t blocks = (plane + 255) / 256;
  if (blocks > (size_t)ups::kNumSMs * 16) blocks = (size_t)ups::kNumSMs * 16;
  ups::prep_image_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(image_hwc, h, w, out_h, out_w, pad_h, pad_w, 1.0 / scale,
                                                                              pixel_means[0], pixel_means[1], pixel_means[2],
                                                                              flip ? 1 : 0, blob);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_label_restore(const long long* src0, const long long* src1, int Hp, int Wp, int h, int w, double fx,
                                    int out_h, int out_w, long long* dst0, long long* dst1, void* stream) {
  if (!src0 || !dst0 || (!src1) != (!dst1)) return UPSNET_E_BADARG;
  if (h <= 0 || w <= 0 || h > Hp || w > Wp || out_h <= 0 || out_w <= 0 || !(fx > 0.0)) return UPSNET_E_BADARG;
  const size_t n = (size_t)out_h * out_w;
  size_t blocks = (n + 255) / 256;
  if (blocks > (size_t)ups::kNumSMs * 8) blocks = (size_t)ups::kNumSMs * 8;
  const dim3 grid((unsigned)blocks, src1 ? 2 : 1);
  ups::label_restore_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(src0, src1, Wp, h, w, 1.0 / fx, out_h, out_w, dst0, dst1);
  UPS_CHECK_LAUNCH();
  return 0;
}
