// detection.cu -- fused device-side detection glue between the hot kernels: RPN box decode for the pre-NMS
// top-k of every pyramid level, and the two halves of MaskROI (candidate selection + ordering + decode before
// the segmented NMS, global top-n + compaction after it).
//
// The reference does this on the HOST in numpy (operators/functions/pyramid_proposal.py:83-131,
// operators/modules/mask_roi.py:36-146, bbox/bbox_transform.py:290-330,45-60); the engine's first GPU version
// restated it with ~30 elementwise / sort / scatter torch launches per call, which made ~600 tiny launches per
// image.  Each kernel here replaces one such cluster with a single launch and keeps the arithmetic order of
// the reference's float32 formulas (separately rounded mul/add: no FMA contraction), so the decoded boxes --
// and therefore every NMS decision -- are the ones the torch restatement (still used on CPU tensors and as the
// test oracle for these kernels) produces.
#include <cfloat>

#include "anchors.cuh"
#include "common.cuh"
#include "cta.cuh"

namespace ups {

// bbox/bbox_transform.py:290-330 for one (box, delta) pair; weights divide the deltas; clip to the image.
__device__ __forceinline__ float4 decode_clip(float x1, float y1, float x2, float y2, float dx, float dy, float dw, float dh,
                                              float xform_clip, float im_h, float im_w) {
  const float w = __fadd_rn(__fsub_rn(x2, x1), 1.0f), h = __fadd_rn(__fsub_rn(y2, y1), 1.0f);
  const float cx = __fadd_rn(x1, __fmul_rn(0.5f, w)), cy = __fadd_rn(y1, __fmul_rn(0.5f, h));
  dw = fminf(dw, xform_clip);
  dh = fminf(dh, xform_clip);
  const float pcx = __fadd_rn(__fmul_rn(dx, w), cx), pcy = __fadd_rn(__fmul_rn(dy, h), cy);
  const float pw = __fmul_rn(expf(dw), w), ph = __fmul_rn(expf(dh), h);
  float4 o;
  o.x = __fsub_rn(pcx, __fmul_rn(0.5f, pw));
  o.y = __fsub_rn(pcy, __fmul_rn(0.5f, ph));
  o.z = __fsub_rn(__fadd_rn(pcx, __fmul_rn(0.5f, pw)), 1.0f);
  o.w = __fsub_rn(__fadd_rn(pcy, __fmul_rn(0.5f, ph)), 1.0f);
  const float mx = __fsub_rn(im_w, 1.0f), my = __fsub_rn(im_h, 1.0f);
  o.x = fminf(fmaxf(o.x, 0.f), mx);
  o.y = fminf(fmaxf(o.y, 0.f), my);
  o.z = fminf(fmaxf(o.z, 0.f), mx);
  o.w = fminf(fmaxf(o.w, 0.f), my);
  return o;
}

// ----------------------------------------------------------------------------------------------
// RPN decode
// ----------------------------------------------------------------------------------------------
constexpr int kMaxLevels = 8;
struct RpnDecodeParams {
  const float* deltas[kMaxLevels];       // [4A, h, w] fp32 (channel = a*4 + c)
  const long long* idx[kMaxLevels];      // [k] flat indices in (y, x, a) order
  int k[kMaxLevels], h[kMaxLevels], w[kMaxLevels], stride[kMaxLevels], start[kMaxLevels + 1];
  const double* base;                    // [L, A, 4] generate_anchors() of every level (float64, like the reference)
  int L, A;
  float im_h, im_w, xform_clip;
  float* out;                            // [sum k, 4]
};

__global__ void rpn_decode_kernel(const RpnDecodeParams p) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= p.start[p.L]) return;
  int l = 0;
  while (l + 1 < p.L && t >= p.start[l + 1]) ++l;
  const long long i = p.idx[l][t - p.start[l]];
  const int a = (int)(i % p.A);
  const long long pix = i / p.A;
  const int x = (int)(pix % p.w[l]), y = (int)(pix / p.w[l]);
  const float4 an = shifted_anchor(p.base + ((size_t)l * p.A + a) * 4, x, y, p.stride[l]);
  const size_t hw = (size_t)p.h[l] * p.w[l];
  const float* d = p.deltas[l] + (size_t)a * 4 * hw + (size_t)y * p.w[l] + x;
  const float4 o = decode_clip(an.x, an.y, an.z, an.w, __ldg(d), __ldg(d + hw), __ldg(d + 2 * hw), __ldg(d + 3 * hw),
                               p.xform_clip, p.im_h, p.im_w);
  reinterpret_cast<float4*>(p.out)[t] = o;
}

// ----------------------------------------------------------------------------------------------
// MaskROI, part 1: candidates -> (segment asc, score desc, index asc) order -> decoded boxes + segment offsets
// ----------------------------------------------------------------------------------------------
constexpr int kSortN = 8192;
constexpr int kMrThreads = 1024;

__global__ void __launch_bounds__(kMrThreads, 1)
maskroi_prepare_kernel(const float* __restrict__ rois, const uint8_t* __restrict__ roi_valid,
                       const float* __restrict__ bbox_delta, const float* __restrict__ cls_prob, int R, int C,
                       int class_agnostic, float score_thresh, float wx, float wy, float ww, float wh, float xform_clip,
                       float im_h, float im_w, float* __restrict__ sc_out, int* __restrict__ cls_out,
                       float* __restrict__ bx_out, int* __restrict__ offs_out) {
  extern __shared__ unsigned long long keys[];   // kSortN
  __shared__ int seg_cnt[130];
  const int Cm = C - 1, n = R * Cm;
  const int nseg = class_agnostic ? 1 : Cm;
  const int tid = threadIdx.x;
  __shared__ int s_ncand;
  for (int s = tid; s <= nseg; s += kMrThreads) seg_cnt[s] = 0;
  if (tid == 0) s_ncand = 0;
  __syncthreads();
  // keys of the CANDIDATES only (their final order is fixed by the sort, so the append order is irrelevant)
  for (int i = tid; i < n; i += kMrThreads) {
    const int r = i / Cm, c = i - r * Cm;
    const float pr = __ldg(cls_prob + (size_t)r * C + c + 1);
    if (pr > score_thresh && roi_valid[r] != 0) {
      const int seg = class_agnostic ? 0 : c;
      // descending score: prob > thresh >= 0 is a positive float, whose bit pattern is monotonic
      const unsigned inv = 0xffffffffu - __float_as_uint(pr);
      keys[atomicAdd(&s_ncand, 1)] = ((unsigned long long)seg << 45) | ((unsigned long long)inv << 13) | (unsigned long long)i;
      atomicAdd(&seg_cnt[seg], 1);
    }
  }
  __syncthreads();
  int sortN = 64;
  while (sortN < s_ncand) sortN <<= 1;
  for (int i = s_ncand + tid; i < sortN; i += kMrThreads) keys[i] = ~0ull;
  __syncthreads();
  cta_bitonic_sort<kMrThreads, false>(keys, sortN);   // ascending, over the next power of two >= the candidate count
  if (tid == 0) {
    int acc = 0;
    for (int s = 0; s < nseg; ++s) { offs_out[s] = acc; acc += seg_cnt[s]; }
    offs_out[nseg] = acc;
    seg_cnt[nseg + 1] = acc;
  }
  __syncthreads();
  const int n_cand = seg_cnt[nseg + 1];
  for (int pidx = tid; pidx < n; pidx += kMrThreads) {
    float sc = -1.0f;
    int cls = 0;
    float4 bx = make_float4(0.f, 0.f, 0.f, 0.f);
    if (pidx < n_cand) {
      const int i = (int)(keys[pidx] & 0x1fffull);
      const int r = i / Cm, c = i - r * Cm;
      cls = c + 1;
      sc = __ldg(cls_prob + (size_t)r * C + cls);
      const float* ro = rois + (size_t)r * 5 + 1;
      const float* d = bbox_delta + (size_t)r * 4 * C + 4 * cls;
      bx = decode_clip(ro[0], ro[1], ro[2], ro[3], __fdiv_rn(d[0], wx), __fdiv_rn(d[1], wy), __fdiv_rn(d[2], ww),
                       __fdiv_rn(d[3], wh), xform_clip, im_h, im_w);
    }
    sc_out[pidx] = sc;
    cls_out[pidx] = cls;
    reinterpret_cast<float4*>(bx_out)[pidx] = bx;
  }
}

// ----------------------------------------------------------------------------------------------
// MaskROI, part 2: NMS survivors (class-major) -> global top-n score threshold -> compaction into `cap` slots
// ----------------------------------------------------------------------------------------------
constexpr int kAllCap = 4096;

__global__ void __launch_bounds__(kMrThreads, 1)
maskroi_finish_kernel(const int* __restrict__ keep, const int* __restrict__ cnt, const int* __restrict__ offs,
                      const float* __restrict__ sc, const int* __restrict__ cls, const float* __restrict__ bx, int nseg,
                      int M, int top_n, int cap, float* __restrict__ out_sc, float* __restrict__ out_bx,
                      long long* __restrict__ out_cls, int* __restrict__ n_out) {
  __shared__ int gidx[kAllCap];
  __shared__ unsigned key[kAllCap];
  __shared__ int seg_base[130];
  __shared__ int warp_sums[kMrThreads / 32];
  const int tid = threadIdx.x;
  const int all_cap = min(nseg * M, kAllCap);
  if (tid == 0) {
    int acc = 0;
    for (int s = 0; s < nseg; ++s) { seg_base[s] = acc; acc += min(max(cnt[s], 0), M); }
    seg_base[nseg] = acc;
  }
  __syncthreads();
  const int nk = min(seg_base[nseg], all_cap);
  // class-major list of survivors (mask_roi.py:96-104), NMS (descending score) order inside a class
  for (int s = 0; s < nseg; ++s) {
    const int b = seg_base[s], c = seg_base[s + 1] - b, o = offs[s];
    for (int j = tid; j < c; j += kMrThreads)
      if (b + j < all_cap) {
        const int g = keep[(size_t)s * M + j] + o;
        gidx[b + j] = g;
        key[b + j] = orderable(sc[g]);
      }
  }
  __syncthreads();
  // k-th largest score (mask_roi.py:106-121): 4-pass radix select over the order-preserving keys
  const int K = min(top_n, all_cap);
  const unsigned kth = (top_n > 0 && nk >= K)
                           ? cta_radix_select<kMrThreads, unsigned, 32, 8, true>([&](int i) { return key[i]; }, nk, K)
                           : 0u;      // keep everything
  // ordered compaction of {score >= kth} into the output slots
  constexpr int PER = kAllCap / kMrThreads;
  int flags[PER], mine = 0;
#pragma unroll
  for (int e = 0; e < PER; ++e) {
    const int i = tid * PER + e;
    flags[e] = (i < nk && key[i] >= kth) ? 1 : 0;
    mine += flags[e];
  }
  int total;
  int dst = cta_scan_excl<kMrThreads>(mine, warp_sums, &total);
  const int n_sel = min(total, cap);
#pragma unroll
  for (int e = 0; e < PER; ++e) {
    if (flags[e]) {
      if (dst < cap) {
        const int g = gidx[tid * PER + e];
        out_sc[dst] = sc[g];
        out_cls[dst] = (long long)cls[g];
        out_bx[(size_t)dst * 5] = 0.f;
        const float4 b4 = reinterpret_cast<const float4*>(bx)[g];
        out_bx[(size_t)dst * 5 + 1] = b4.x; out_bx[(size_t)dst * 5 + 2] = b4.y;
        out_bx[(size_t)dst * 5 + 3] = b4.z; out_bx[(size_t)dst * 5 + 4] = b4.w;
      }
      ++dst;
    }
  }
  for (int sidx = n_sel + tid; sidx < cap; sidx += kMrThreads) {
    out_sc[sidx] = (sidx == 0) ? 1.0f : 0.f;     // mask_roi.py:132-139: nothing survives -> one dummy detection
    out_cls[sidx] = 0;
#pragma unroll
    for (int e = 0; e < 5; ++e) out_bx[(size_t)sidx * 5 + e] = 0.f;
  }
  if (tid == 0) {
    n_out[0] = n_sel == 0 ? 1 : n_sel;
    // truncation flags (the reference keeps every survivor / every box tied at the top-n threshold, mask_roi.py:96-121):
    // bit 0: more NMS survivors than the kAllCap candidate slots (the tail of the class-major list was not considered),
    // bit 1: more boxes at or above the top-n threshold than the `cap` output slots (the surplus of the tie was dropped)
    n_out[1] = (seg_base[nseg] > all_cap ? 1 : 0) | (total > cap ? 2 : 0);
  }
}

}  // namespace ups

extern "C" int upsnet_rpn_decode(const float* const* deltas, const long long* const* top_idx, const int* k, const int* hs,
                                 const int* ws, const int* strides, const double* base_anchors, int L, int A, float im_h,
                                 float im_w, float* boxes_out, void* stream) {
  if (!deltas || !top_idx || !k || !hs || !ws || !strides || !base_anchors || !boxes_out) return UPSNET_E_BADARG;
  if (L <= 0 || L > ups::kMaxLevels || A <= 0) return UPSNET_E_BADARG;
  ups::RpnDecodeParams p{};
  int acc = 0;
  for (int l = 0; l < L; ++l) {
    if (k[l] < 0 || hs[l] <= 0 || ws[l] <= 0 || (k[l] > 0 && (!deltas[l] || !top_idx[l]))) return UPSNET_E_BADARG;
    p.deltas[l] = deltas[l]; p.idx[l] = top_idx[l];
    p.k[l] = k[l]; p.h[l] = hs[l]; p.w[l] = ws[l]; p.stride[l] = strides[l];
    p.start[l] = acc;
    acc += k[l];
  }
  p.start[L] = acc;
  p.base = base_anchors; p.L = L; p.A = A; p.im_h = im_h; p.im_w = im_w;
  p.xform_clip = (float)4.135166556742356;   // log(1000 / 16), bbox_transform.py
  p.out = boxes_out;
  if (acc == 0) return 0;
  ups::rpn_decode_kernel<<<(acc + 255) / 256, 256, 0, (cudaStream_t)stream>>>(p);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_maskroi_prepare(const float* rois, const unsigned char* roi_valid, const float* bbox_delta,
                                      const float* cls_prob, int R, int C, int class_agnostic, float score_thresh,
                                      const float weights[4], float im_h, float im_w, float* sc_out, int* cls_out,
                                      float* bx_out, int* offs_out, void* stream) {
  if (!rois || !roi_valid || !bbox_delta || !cls_prob || !weights || !sc_out || !cls_out || !bx_out || !offs_out)
    return UPSNET_E_BADARG;
  if (R <= 0 || C < 2) return UPSNET_E_BADARG;
  if ((long long)R * (C - 1) > ups::kSortN || C - 1 > 128 || score_thresh < 0.f) return UPSNET_E_UNSUPPORTED;
  static ups::PerDeviceOnce configured;
  if (configured.need()) {
    UPS_CUDA(cudaFuncSetAttribute(ups::maskroi_prepare_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  ups::kSortN * 8));
  }
  ups::maskroi_prepare_kernel<<<1, ups::kMrThreads, ups::kSortN * 8, (cudaStream_t)stream>>>(
      rois, roi_valid, bbox_delta, cls_prob, R, C, class_agnostic, score_thresh, weights[0], weights[1], weights[2],
      weights[3], (float)4.135166556742356, im_h, im_w, sc_out, cls_out, bx_out, offs_out);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_maskroi_finish(const int* keep, const int* keep_cnt, const int* seg_offsets, const float* sc,
                                     const int* cls, const float* bx, int nseg, int max_seg_len, int top_n, int cap,
                                     float* out_sc, float* out_bx, long long* out_cls, int* n_out, void* stream) {
  if (!keep || !keep_cnt || !seg_offsets || !sc || !cls || !bx || !out_sc || !out_bx || !out_cls || !n_out)
    return UPSNET_E_BADARG;
  if (nseg <= 0 || nseg > 128 || max_seg_len <= 0 || cap <= 0 || top_n < 0) return UPSNET_E_BADARG;
  ups::maskroi_finish_kernel<<<1, ups::kMrThreads, 0, (cudaStream_t)stream>>>(
      keep, keep_cnt, seg_offsets, sc, cls, bx, nseg, max_seg_len, top_n, cap, out_sc, out_bx, out_cls, n_out);
  UPS_CHECK_LAUNCH();
  return 0;
}

// ----------------------------------------------------------------------------------------------
// RPN pre-NMS top-k for all pyramid levels (pyramid_proposal.py:104-118: argsort(-scores)[:pre_nms_top_n]).
//
// Exact radix select on the 54-bit key  (orderable(score) << 22) | (2^22-1 - flat_index):  all keys are
// distinct, so "the k largest" is a unique set and ties in the score resolve to the lowest (y,x,a) index --
// a valid instance of the reference's unspecified tie order.  Five digit passes (11+11+10 score bits, 11+11
// index bits): every CTA histograms its slice of the level in shared memory, the LAST CTA of a level to
// finish (ticket) scans the 2048 bins, fixes the digit and re-arms the counters, so a pass is one launch for
// all levels.  Then one gather of the keys >= k-th key and one single-CTA bitonic sort per level.
// ----------------------------------------------------------------------------------------------
namespace ups {

constexpr int kTkBins = 2048, kTkThreads = 512, kTkItems = 8, kTkMaxK = 2048, kTkIdxBits = 22;

struct TopkLevel {
  const float* prob;      // [A, h, w]
  int hw, L, k, blocks;   // L = A*hw elements, k = min(pre_nms_top_n, L)
  int out_start;          // offset of this level in the concatenated outputs
};
struct TopkParams {
  TopkLevel lv[kMaxLevels];
  int nlev, A;
  unsigned int* hist;            // [nlev][kTkBins]
  unsigned int* ticket;          // [nlev]
  unsigned long long* prefix;    // [nlev]  key bits fixed so far
  int* need;                     // [nlev]  how many of the k are still to be found inside the current prefix
  unsigned int* fill;            // [nlev]  gather cursor
  int* done;                     // [nlev]  set once the bucket of the current prefix is small enough to be sorted whole
  unsigned long long* keys;      // [nlev][kTkMaxK]
  float* out_scores; long long* out_idx;
};

__device__ __forceinline__ unsigned long long topk_key(float s, unsigned int flat) {
  return ((unsigned long long)orderable(s) << kTkIdxBits) | (unsigned long long)((1u << kTkIdxBits) - 1u - flat);
}
// element e of the [A,h,w] array -> flat (y,x,a) index
__device__ __forceinline__ unsigned int topk_flat(int e, int hw, int A) {
  const int a = e / hw, pix = e - a * hw;
  return (unsigned int)(pix * A + a);
}

// pass over digit [shift, shift+bits): mask_hi selects the already fixed (higher) bits
__global__ void __launch_bounds__(kTkThreads)
topk_pass_kernel(const TopkParams p, int shift, int bits, int first) {
  const int l = blockIdx.y;
  const TopkLevel lv = p.lv[l];
  if ((int)blockIdx.x >= lv.blocks) return;
  if (!first && p.done[l]) return;      // an earlier pass already narrowed the candidates to what the sort kernel can take
  __shared__ unsigned int sh[kTkBins];
  for (int b = threadIdx.x; b < kTkBins; b += kTkThreads) sh[b] = 0;
  __syncthreads();
  const unsigned long long fixed = first ? 0ull : p.prefix[l];
  const unsigned long long mask_hi = first ? 0ull : (~0ull << (shift + bits));
  const unsigned int dmask = (1u << bits) - 1u;
  const int e0 = blockIdx.x * (kTkThreads * kTkItems);
#pragma unroll 4
  for (int it = 0; it < kTkItems; ++it) {
    const int e = e0 + it * kTkThreads + threadIdx.x;
    bool act = false;
    unsigned int bin = 0xffffffffu;
    if (e < lv.L) {
      const unsigned long long key = topk_key(__ldg(lv.prob + e), topk_flat(e, lv.hw, p.A));
      act = (key & mask_hi) == fixed;
      if (act) bin = (unsigned int)(key >> shift) & dmask;
    }
    // scores cluster in a handful of exponent bins (first pass) or tie exactly (saturated sigmoid): aggregate equal
    // bins inside the warp so that one lane issues one shared-memory atomic per distinct bin
    const unsigned int peers = __match_any_sync(0xffffffffu, bin);
    if (act && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&sh[bin], (unsigned int)__popc(peers));
  }
  __syncthreads();
  unsigned int* gh = p.hist + (size_t)l * kTkBins;
  for (int b = threadIdx.x; b < kTkBins; b += kTkThreads)
    if (sh[b]) atomicAdd(&gh[b], sh[b]);
  if (!last_cta(&p.ticket[l], (unsigned)lv.blocks)) return;
  // ---- last CTA of this level: find the digit that contains the need-th largest key ----
  for (int b = threadIdx.x; b < kTkBins; b += kTkThreads) { sh[b] = __ldcg(&gh[b]); gh[b] = 0; }
  __syncthreads();
  RadixDigit d;
  if (threadIdx.x < 32 && warp_radix_digit<kTkBins, true>(sh, first ? lv.k : p.need[l], &d)) {
    p.need[l] = d.need;
    p.prefix[l] = fixed | ((unsigned long long)d.digit << shift);
    // early exit: everything above the bucket (k - need') plus the WHOLE bucket fits the sort buffer -> no need to
    // resolve the remaining digits, the sort orders the bucket and the first k are taken
    if ((long long)(lv.k - d.need) + (long long)sh[d.digit] <= (long long)kTkMaxK) p.done[l] = 1;
    p.ticket[l] = 0;
    p.fill[l] = 0;
  }
}

__global__ void __launch_bounds__(kTkThreads)
topk_gather_kernel(const TopkParams p) {
  const int l = blockIdx.y;
  const TopkLevel lv = p.lv[l];
  if ((int)blockIdx.x >= lv.blocks) return;
  const unsigned long long kth = p.prefix[l];
  const int e0 = blockIdx.x * (kTkThreads * kTkItems);
  for (int it = 0; it < kTkItems; ++it) {
    const int e = e0 + it * kTkThreads + threadIdx.x;
    if (e < lv.L) {
      const unsigned long long key = topk_key(__ldg(lv.prob + e), topk_flat(e, lv.hw, p.A));
      if (key >= kth) {
        const unsigned int pos = atomicAdd(&p.fill[l], 1u);
        if (pos < (unsigned int)kTkMaxK) p.keys[(size_t)l * kTkMaxK + pos] = key;
      }
    }
  }
}

__global__ void __launch_bounds__(1024)
topk_sort_kernel(const TopkParams p) {
  const int l = blockIdx.x;
  const TopkLevel lv = p.lv[l];
  __shared__ unsigned long long sk[kTkMaxK];
  const int tid = threadIdx.x;
  const int nk = min((int)p.fill[l], kTkMaxK);       // == k unless a pass exited early with a whole bucket
  for (int i = tid; i < kTkMaxK; i += 1024) sk[i] = i < nk ? p.keys[(size_t)l * kTkMaxK + i] : 0ull;
  __syncthreads();
  cta_bitonic_sort<1024, true>(sk, kTkMaxK);
  for (int i = tid; i < lv.k; i += 1024) {
    const unsigned long long key = sk[i];
    p.out_scores[lv.out_start + i] = from_orderable((unsigned int)(key >> kTkIdxBits));
    p.out_idx[lv.out_start + i] = (long long)((1u << kTkIdxBits) - 1u - (unsigned int)(key & ((1u << kTkIdxBits) - 1u)));
  }
}

inline size_t topk_layout(int L, void* base, TopkParams& p) {
  WsCarve c(base);
  p.hist = c.take<unsigned int>((size_t)L * kTkBins);
  p.keys = c.take<unsigned long long>((size_t)L * kTkMaxK);
  p.prefix = c.take<unsigned long long>(L);
  // ticket, need, fill and done share one region, so that one memset clears them
  unsigned int* ctr = c.take<unsigned int>((size_t)L * 4);
  if (ctr) {
    p.ticket = ctr; p.need = (int*)(ctr + L); p.fill = ctr + 2 * L; p.done = (int*)(ctr + 3 * L);
  }
  return c.bytes();
}

}  // namespace ups

extern "C" int upsnet_rpn_topk_workspace_bytes(int L, size_t* bytes) {
  if (!bytes || L <= 0 || L > ups::kMaxLevels) return UPSNET_E_BADARG;
  ups::TopkParams p{};
  *bytes = ups::topk_layout(L, nullptr, p);
  return 0;
}

extern "C" int upsnet_rpn_topk(const float* const* probs, const int* hs, const int* ws, int L, int A, int pre_nms_top_n,
                               float* out_scores, long long* out_idx, void* workspace, size_t workspace_bytes,
                               void* stream) {
  using namespace ups;
  if (!probs || !hs || !ws || !out_scores || !out_idx || !workspace) return UPSNET_E_BADARG;
  if (L <= 0 || L > kMaxLevels || A <= 0 || pre_nms_top_n <= 0) return UPSNET_E_BADARG;
  if (pre_nms_top_n > kTkMaxK) return UPSNET_E_UNSUPPORTED;
  TopkParams p{};
  if (workspace_bytes < topk_layout(L, workspace, p)) return UPSNET_E_WORKSPACE;
  p.nlev = L; p.A = A; p.out_scores = out_scores; p.out_idx = out_idx;
  int acc = 0, max_blocks = 0;
  for (int l = 0; l < L; ++l) {
    if (!probs[l] || hs[l] <= 0 || ws[l] <= 0) return UPSNET_E_BADARG;
    const long long Ll = (long long)A * hs[l] * ws[l];
    if (Ll >= (1ll << kTkIdxBits)) return UPSNET_E_UNSUPPORTED;
    p.lv[l].prob = probs[l]; p.lv[l].hw = hs[l] * ws[l]; p.lv[l].L = (int)Ll;
    p.lv[l].k = (int)(Ll < pre_nms_top_n ? Ll : pre_nms_top_n);
    p.lv[l].blocks = (int)((Ll + kTkThreads * kTkItems - 1) / (kTkThreads * kTkItems));
    p.lv[l].out_start = acc;
    acc += p.lv[l].k;
    if (p.lv[l].blocks > max_blocks) max_blocks = p.lv[l].blocks;
  }
  cudaStream_t st = (cudaStream_t)stream;
  // histograms + tickets start at zero (every pass re-arms them for the next one)
  UPS_CUDA(cudaMemsetAsync(p.hist, 0, (size_t)L * kTkBins * 4, st));
  UPS_CUDA(cudaMemsetAsync(p.ticket, 0, (size_t)L * 4 * 4, st));    // ticket, need, fill, done
  const dim3 grid((unsigned)max_blocks, (unsigned)L);
  const int shifts[5] = {43, 32, 22, 11, 0}, nbits[5] = {11, 11, 10, 11, 11};
  for (int ps = 0; ps < 5; ++ps) {
    topk_pass_kernel<<<grid, kTkThreads, 0, st>>>(p, shifts[ps], nbits[ps], ps == 0 ? 1 : 0);
    UPS_CHECK_LAUNCH();
  }
  topk_gather_kernel<<<grid, kTkThreads, 0, st>>>(p);
  UPS_CHECK_LAUNCH();
  topk_sort_kernel<<<L, 1024, 0, st>>>(p);
  UPS_CHECK_LAUNCH();
  return 0;
}

// ----------------------------------------------------------------------------------------------
// RPN post-NMS collect (operators/modules/pyramid_proposal.py:61-67 + functions/pyramid_proposal.py:196-222):
// the first min(cnt, post) NMS survivors of every level, then the `post` best of their union by score, as
// fixed-size outputs (rois [post,5] with zero rows past the live count, scores, validity flags).
// One CTA: 45-bit keys (orderable(score) << 13 | 8191 - position in the level-major candidate list) in shared
// memory, 4-pass radix select of the post-th largest, compaction, bitonic sort of the selected <= 2048 keys.
// ----------------------------------------------------------------------------------------------
namespace ups {

constexpr int kColMaxCand = 8192, kColMaxPost = 2048;

__global__ void __launch_bounds__(1024, 1)
rpn_collect_kernel(const int* __restrict__ keep, const int* __restrict__ cnt, const int* __restrict__ offs,
                   const float* __restrict__ boxes, const float* __restrict__ scores, int S, int max_len, int post,
                   float* __restrict__ rois, float* __restrict__ out_scores, unsigned char* __restrict__ ok) {
  extern __shared__ unsigned long long ck[];            // [kColMaxCand] candidate keys, then [kColMaxPost] selected
  unsigned long long* sel = ck + kColMaxCand;
  __shared__ int seg_base[kMaxLevels + 1];
  __shared__ int s_nsel;
  const int tid = threadIdx.x;
  if (tid == 0) {
    int acc = 0;
    for (int s = 0; s < S; ++s) { seg_base[s] = acc; acc += min(min(max(cnt[s], 0), max_len), post); }
    seg_base[S] = min(acc, kColMaxCand);
    s_nsel = 0;
  }
  __syncthreads();
  const int C = seg_base[S];
  for (int s = 0; s < S; ++s) {
    const int b = seg_base[s], n = min(seg_base[s + 1], kColMaxCand) - b, o = offs[s];
    for (int j = tid; j < n; j += 1024) {
      const int g = keep[(size_t)s * max_len + j] + o;
      ck[b + j] = ((unsigned long long)orderable(scores[g]) << 13) | (unsigned long long)(8191 - (b + j));
    }
  }
  __syncthreads();
  const unsigned long long kth =
      C > post ? cta_radix_select<1024, unsigned long long, 45, 12, true>([&](int i) { return ck[i]; }, C, post) : 0ull;
  // selected keys (all distinct): exactly min(C, post) of them; order fixed by the sort below
  for (int i = tid; i < C; i += 1024)
    if (ck[i] >= kth) {
      const int pos = atomicAdd(&s_nsel, 1);
      if (pos < kColMaxPost) sel[pos] = ck[i];
    }
  __syncthreads();
  const int nsel = min(s_nsel, min(post, kColMaxPost));
  int sortN = 64;
  while (sortN < nsel) sortN <<= 1;
  for (int i = nsel + tid; i < sortN; i += 1024) sel[i] = 0ull;
  __syncthreads();
  cta_bitonic_sort<1024, true>(sel, sortN);
  for (int i = tid; i < post; i += 1024) {
    float4 bx = make_float4(0.f, 0.f, 0.f, 0.f);
    float sc = 0.f;
    unsigned char live = 0;
    if (i < nsel) {
      const int fp = 8191 - (int)(sel[i] & 8191ull);
      int s = 0;
      while (s + 1 < S && fp >= seg_base[s + 1]) ++s;
      const int g = keep[(size_t)s * max_len + (fp - seg_base[s])] + offs[s];
      bx = reinterpret_cast<const float4*>(boxes)[g];
      sc = scores[g];
      live = 1;
    }
    rois[(size_t)i * 5] = 0.f;
    rois[(size_t)i * 5 + 1] = bx.x; rois[(size_t)i * 5 + 2] = bx.y;
    rois[(size_t)i * 5 + 3] = bx.z; rois[(size_t)i * 5 + 4] = bx.w;
    out_scores[i] = sc;
    ok[i] = live;
  }
}

}  // namespace ups

extern "C" int upsnet_rpn_collect(const int* keep, const int* keep_cnt, const int* seg_offsets, const float* boxes,
                                  const float* scores, int S, int max_seg_len, int post_nms_top_n, float* rois,
                                  float* out_scores, unsigned char* valid, void* stream) {
  using namespace ups;
  if (!keep || !keep_cnt || !seg_offsets || !boxes || !scores || !rois || !out_scores || !valid) return UPSNET_E_BADARG;
  if (S <= 0 || S > kMaxLevels || max_seg_len <= 0 || post_nms_top_n <= 0) return UPSNET_E_BADARG;
  if (post_nms_top_n > kColMaxPost || (long long)S * (max_seg_len < post_nms_top_n ? max_seg_len : post_nms_top_n) > kColMaxCand)
    return UPSNET_E_UNSUPPORTED;
  if (((uintptr_t)boxes) & 15) return UPSNET_E_BADARG;
  const size_t smem = (size_t)(kColMaxCand + kColMaxPost) * 8;
  static ups::PerDeviceOnce configured;
  if (configured.need()) {
    UPS_CUDA(cudaFuncSetAttribute(rpn_collect_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  rpn_collect_kernel<<<1, 1024, smem, (cudaStream_t)stream>>>(keep, keep_cnt, seg_offsets, boxes, scores, S, max_seg_len,
                                                               post_nms_top_n, rois, out_scores, valid);
  UPS_CHECK_LAUNCH();
  return 0;
}

// ----------------------------------------------------------------------------------------------
// Mask-branch row plan.  The branch maps a box (batch index + 4 coordinates) to its logits with no dependence on the
// other rows, so the panoptic candidates whose box is bit-identical to a detection's box reuse that detection's row:
//   rows [0, n1)  = the detections, in order;  rows [n1, u) = the candidates that match no detection, in order;
//   pan_row[j]    = the row candidate j's logits come from (0 for j >= n2);  rows [u, cap1 + cap2) are zeroed.
// One CTA, candidates in chunks of the block: ballot + per-warp counts keep the candidate order (deterministic).
// ----------------------------------------------------------------------------------------------
namespace ups {

constexpr int kRowThreads = 128;

__global__ void __launch_bounds__(kRowThreads)
mask_rows_kernel(const float* __restrict__ b1, const int* __restrict__ n1p, int cap1, const float* __restrict__ b2,
                 const int* __restrict__ n2p, int cap2, float* __restrict__ rows, int* __restrict__ u_out,
                 int* __restrict__ pan_row) {
  __shared__ int s_cnt[kRowThreads / 32];
  const int n1 = min(max(*n1p, 0), cap1), n2 = min(max(*n2p, 0), cap2);
  const int tid = threadIdx.x;
  const uint32_t* d = reinterpret_cast<const uint32_t*>(b1);
  for (int k = tid; k < n1 * 5; k += kRowThreads) rows[k] = b1[k];
  int base = n1;
  for (int j0 = 0; j0 < cap2; j0 += kRowThreads) {
    const int j = j0 + tid;
    int src = 0;
    bool fresh = false;
    if (j < n2) {
      const uint32_t* c = reinterpret_cast<const uint32_t*>(b2) + (size_t)j * 5;
      const uint32_t c0 = c[0], c1 = c[1], c2 = c[2], c3 = c[3], c4 = c[4];
      src = -1;
      for (int i = 0; i < n1; ++i) {
        const uint32_t* e = d + (size_t)i * 5;
        if (e[0] == c0 && e[1] == c1 && e[2] == c2 && e[3] == c3 && e[4] == c4) { src = i; break; }
      }
      fresh = src < 0;
    }
    int tot;
    const int rank = cta_ballot_rank<kRowThreads>(fresh, s_cnt, &tot);
    if (fresh) {
      src = base + rank;
      for (int k = 0; k < 5; ++k) rows[(size_t)src * 5 + k] = b2[(size_t)j * 5 + k];
    }
    if (j < cap2) pan_row[j] = src;
    base += tot;
  }
  for (int k = base * 5 + tid; k < (cap1 + cap2) * 5; k += kRowThreads) rows[k] = 0.f;
  if (tid == 0) *u_out = base;
}

}  // namespace ups

extern "C" int upsnet_mask_rows(const float* b1, const int* n1, int cap1, const float* b2, const int* n2, int cap2,
                                float* rows, int* u, int* pan_row, void* stream) {
  if (!b1 || !n1 || !b2 || !n2 || !rows || !u || !pan_row || cap1 <= 0 || cap2 <= 0) return UPSNET_E_BADARG;
  if ((long long)cap1 + cap2 > (1 << 20)) return UPSNET_E_UNSUPPORTED;
  ups::mask_rows_kernel<<<1, ups::kRowThreads, 0, (cudaStream_t)stream>>>(b1, n1, cap1, b2, n2, cap2, rows, u, pan_row);
  UPS_CHECK_LAUNCH();
  return 0;
}
