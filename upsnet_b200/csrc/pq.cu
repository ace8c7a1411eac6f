// pq.cu -- panoptic quality statistics of one image (SURVEY section 8f row f4, evaluation half), device resident:
//
//  * upsnet_pq_update: dataset/base_dataset.py:462-511 _converter_2ch_single_core (2-channel map -> segments) composed
//    with :513-608 _pq_compute_single_core (the (gt, prediction) confusion counts, IoU > 0.5 matching, FN with crowd
//    bookkeeping, FP with the VOID + crowd ignore rule).  Reference: numpy on the host, np.unique over the 2-channel map,
//    one full-image mask per segment, then np.unique over a 2 M-element uint64 pair map.
//    Here: one pixel pass that counts (gt slot, prediction segment) pairs in a per-block shared hash with
//    warp-aggregated inserts, flushed to a global hash; then one CTA that does matching, FN, crowd lookup and FP and adds
//    to the per-category accumulator.  HBM-bound: 6 bytes per pixel.
#include "common.cuh"

namespace ups {

constexpr int kPqMaxGt = UPSNET_PQ_MAX_GT;
constexpr int kPqMaxPairs = UPSNET_PQ_MAX_PAIRS;
constexpr int kPqHashBits = 17;                  // global pair hash: 2 * kPqMaxPairs slots, load <= 1/2
constexpr int kPqHash = 1 << kPqHashBits;
constexpr int kPqLocalBits = 11;                 // per-block shared pair hash
constexpr int kPqLocal = 1 << kPqLocalBits;
constexpr int kPqMaxPred = UPSNET_PQ_MAX_PRED;
constexpr int kPqPredBits = 12;                  // finalize: prediction-segment hash, load <= 1/2
constexpr int kPqPred = 1 << kPqPredBits;
constexpr int kPqFinThreads = 1024;
constexpr unsigned kPqEmpty = 0xffffffffu;
// gt slots: 0..G-1 = rows of the (id-sorted) table, then VOID (id 0) and "id not in the table".  A pair key is
// slot << 16 | prediction key, the prediction key class << 8 | instance (instance 0 for stuff classes).
constexpr unsigned kSlotVoid = kPqMaxGt, kSlotUnknown = kPqMaxGt + 1;
static_assert(((kSlotUnknown << 16) | 0xffffu) < kPqEmpty, "pair keys must not collide with the empty marker");

struct PqWs {
  unsigned* keys;   // [kPqHash] pair key or kPqEmpty
  unsigned* cnt;    // [kPqHash] pixel count of the pair
  int* n_pairs;     // [1] distinct pairs inserted
  unsigned* list;   // [kPqMaxPairs] hash slot of the i-th inserted pair
};

static size_t pq_ws_layout(PqWs* ws, char* base) {
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = align_up(off + bytes, 256); return o; };
  const size_t o_keys = take(sizeof(unsigned) * kPqHash), o_cnt = take(sizeof(unsigned) * kPqHash);
  const size_t o_n = take(sizeof(int)), o_list = take(sizeof(unsigned) * kPqMaxPairs);
  if (ws) {
    ws->keys = (unsigned*)(base + o_keys); ws->cnt = (unsigned*)(base + o_cnt);
    ws->n_pairs = (int*)(base + o_n); ws->list = (unsigned*)(base + o_list);
  }
  return off;
}

__device__ __forceinline__ unsigned pq_hash(unsigned key, int bits) { return (key * 2654435761u) >> (32 - bits); }

__device__ void pq_global_insert(const PqWs& ws, unsigned key, unsigned c, int* err) {
  unsigned h = pq_hash(key, kPqHashBits);
  for (int probe = 0; probe < kPqHash; ++probe) {
    unsigned prev = ws.keys[h];
    if (prev == kPqEmpty) {
      if (*(volatile int*)ws.n_pairs >= kPqMaxPairs) break;   // over the cap: the result is invalid anyway
      prev = atomicCAS(ws.keys + h, kPqEmpty, key);
      if (prev == kPqEmpty) {
        const int i = atomicAdd(ws.n_pairs, 1);
        if (i < kPqMaxPairs) ws.list[i] = h;
        else break;
      }
    }
    if (prev == kPqEmpty || prev == key) { atomicAdd(ws.cnt + h, c); return; }
    h = (h + 1) & (kPqHash - 1);
  }
  atomicOr(err, UPSNET_PQ_E_PAIRS);
}

__device__ __forceinline__ bool pq_local_insert(unsigned* s_key, unsigned* s_cnt, unsigned key, unsigned c) {
  unsigned h = pq_hash(key, kPqLocalBits);
  for (int probe = 0; probe < 32; ++probe) {
    const unsigned prev = atomicCAS(s_key + h, kPqEmpty, key);
    if (prev == kPqEmpty || prev == key) { atomicAdd(s_cnt + h, c); return true; }
    h = (h + 1) & (kPqLocal - 1);
  }
  return false;
}

__device__ __forceinline__ unsigned byte_of(const unsigned (&w)[3], int b) { return (w[b >> 2] >> ((b & 3) * 8)) & 0xffu; }

// Pixel pass: 4 pixels per thread per step (three 32-bit loads from each map when aligned).  Equal keys of a thread's
// 4 pixels merge into runs; the lanes of a warp holding the same run key elect one leader that adds the run lengths
// (__match_any_sync + __reduce_add_sync, as uni_hist_kernel does with __popc).
__global__ void __launch_bounds__(256)
pq_pixel_kernel(const unsigned char* __restrict__ pan, const unsigned char* __restrict__ gt, size_t HW,
                const long long* __restrict__ table, int G, const unsigned char* __restrict__ cat_flags, PqWs ws, int* err) {
  __shared__ unsigned s_key[kPqLocal], s_cnt[kPqLocal];
  __shared__ int s_ids[kPqMaxGt];
  __shared__ unsigned char s_flags[256];
  __shared__ int s_bad;
  if (G > kPqMaxGt) return;                         // flagged by pq_finalize_kernel
  for (int t = threadIdx.x; t < kPqLocal; t += blockDim.x) { s_key[t] = kPqEmpty; s_cnt[t] = 0; }
  for (int t = threadIdx.x; t < G; t += blockDim.x) s_ids[t] = (int)table[t];
  for (int t = threadIdx.x; t < 256; t += blockDim.x) s_flags[t] = cat_flags[t];
  if (threadIdx.x == 0) s_bad = 0;
  __syncthreads();
  const bool vec = ((reinterpret_cast<uintptr_t>(pan) | reinterpret_cast<uintptr_t>(gt)) & 3) == 0;
  const size_t nq = (HW + 3) / 4;
  int last_id = 0;
  unsigned last_slot = kSlotVoid;
  bool bad = false;
  for (size_t q0 = (size_t)blockIdx.x * blockDim.x; q0 < nq; q0 += (size_t)gridDim.x * blockDim.x) {
    const size_t q = q0 + threadIdx.x;
    unsigned key[4] = {kPqEmpty, kPqEmpty, kPqEmpty, kPqEmpty};
    if (q < nq) {
      unsigned pw[3] = {0u, 0u, 0u}, gw[3] = {0u, 0u, 0u};
      int np = 4;
      if (vec && 4 * q + 4 <= HW) {
        const unsigned* p32 = reinterpret_cast<const unsigned*>(pan + 12 * q);
        const unsigned* g32 = reinterpret_cast<const unsigned*>(gt + 12 * q);
#pragma unroll
        for (int i = 0; i < 3; ++i) { pw[i] = __ldg(p32 + i); gw[i] = __ldg(g32 + i); }
      } else {
        np = (int)min((size_t)4, HW - 4 * q);
#pragma unroll
        for (int b = 0; b < 12; ++b) {
          if (b >= 3 * np) break;
          pw[b >> 2] |= (unsigned)pan[12 * q + b] << ((b & 3) * 8);
          gw[b >> 2] |= (unsigned)gt[12 * q + b] << ((b & 3) * 8);
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (j >= np) break;
        const unsigned cls = byte_of(pw, 3 * j);
        if (cls == 255u) continue;                                  // void prediction: no segment
        const unsigned fl = s_flags[cls];
        if (!(fl & 1u)) { bad = true; continue; }
        const unsigned pk = (cls << 8) | ((fl & 2u) ? byte_of(pw, 3 * j + 1) : 0u);
        const int gid = (int)(byte_of(gw, 3 * j) | (byte_of(gw, 3 * j + 1) << 8) | (byte_of(gw, 3 * j + 2) << 16));
        if (gid != 0 && gid != last_id) {                         // neighbouring pixels nearly always share the id
          int lo = 0, hi = G;                                       // first id >= gid
          while (lo < hi) { const int mid = (lo + hi) >> 1; if (s_ids[mid] < gid) lo = mid + 1; else hi = mid; }
          last_slot = (lo < G && s_ids[lo] == gid) ? (unsigned)lo : kSlotUnknown;
          last_id = gid;
        }
        const unsigned slot = gid == 0 ? kSlotVoid : last_slot;
        key[j] = (slot << 16) | pk;
      }
    }
    // runs of equal keys: the run starting at pixel j has key rk[j] and length rc[j] (all indices static: no local memory)
    unsigned rk[4], rc[4];
    rc[3] = 1u;
#pragma unroll
    for (int j = 2; j >= 0; --j) rc[j] = key[j + 1] == key[j] ? rc[j + 1] + 1u : 1u;
#pragma unroll
    for (int j = 0; j < 4; ++j) rk[j] = (j == 0 || key[j - 1] != key[j]) ? key[j] : kPqEmpty;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (!__any_sync(0xffffffffu, rk[j] != kPqEmpty)) continue;
      const unsigned peers = __match_any_sync(0xffffffffu, rk[j]);
      const unsigned sum = __reduce_add_sync(peers, rc[j]);
      if (rk[j] != kPqEmpty && (int)(__ffs(peers) - 1) == (int)(threadIdx.x & 31))
        if (!pq_local_insert(s_key, s_cnt, rk[j], sum)) pq_global_insert(ws, rk[j], sum, err);
    }
  }
  if (bad) s_bad = 1;
  __syncthreads();
  for (int t = threadIdx.x; t < kPqLocal; t += blockDim.x)
    if (s_key[t] != kPqEmpty) pq_global_insert(ws, s_key[t], s_cnt[t], err);
  if (threadIdx.x == 0 && s_bad) atomicOr(err, UPSNET_PQ_E_PRED_CATEGORY);
}

struct PqFinSmem {
  unsigned pkey[kPqPred], parea[kPqPred], pvoid[kPqPred], pcrowd[kPqPred];
  unsigned mkey[kPqMaxGt];
  double miou[kPqMaxGt];
  double iou[256];
  unsigned short perm[kPqMaxGt];
  int crowd_ord[256], crowd_slot[256], tp[256], fp[256], fn[256];
  unsigned char pmatched[kPqPred], gmatched[kPqMaxGt];
  int n_match, n_pred, err;
};

__device__ int pq_pred_slot(PqFinSmem& s, unsigned pk, bool insert) {
  unsigned h = pq_hash(pk, kPqPredBits);
  for (int probe = 0; probe < kPqPred; ++probe) {
    unsigned prev = s.pkey[h];
    if (prev == kPqEmpty && insert) {
      prev = atomicCAS(s.pkey + h, kPqEmpty, pk);
      if (prev == kPqEmpty) {
        if (atomicAdd(&s.n_pred, 1) >= kPqMaxPred) atomicOr(&s.err, UPSNET_PQ_E_PRED_COUNT);
        return (int)h;
      }
    }
    if (prev == pk) return (int)h;
    if (prev == kPqEmpty) return -1;
    h = (h + 1) & (kPqPred - 1);
  }
  if (insert) atomicOr(&s.err, UPSNET_PQ_E_PRED_COUNT);
  return -1;
}

// One CTA per image: base_dataset.py:544-606 on the pair list.  Matches are collected, ranked by pair key (= ascending
// gt id, then prediction segment: np.unique's order) and their IoUs summed by one thread in that order, so the
// accumulator is bit-identical from run to run.
__global__ void __launch_bounds__(kPqFinThreads)
pq_finalize_kernel(const long long* __restrict__ table, int G, PqWs ws, long long* __restrict__ acc, double* __restrict__ acc_iou,
                   int* err) {
  extern __shared__ __align__(16) unsigned char pq_smem[];
  PqFinSmem& s = *reinterpret_cast<PqFinSmem*>(pq_smem);
  const int tid = threadIdx.x;
  if (G > kPqMaxGt) { if (tid == 0) atomicOr(err, UPSNET_PQ_E_GT_COUNT); return; }
  const long long *t_id = table, *t_cat = table + G, *t_crowd = table + 2 * (size_t)G, *t_area = table + 3 * (size_t)G,
                  *t_ord = table + 4 * (size_t)G;
  for (int t = tid; t < kPqPred; t += blockDim.x) { s.pkey[t] = kPqEmpty; s.parea[t] = 0; s.pvoid[t] = 0; s.pcrowd[t] = 0; s.pmatched[t] = 0; }
  for (int t = tid; t < kPqMaxGt; t += blockDim.x) s.gmatched[t] = 0;
  for (int t = tid; t < 256; t += blockDim.x) {
    s.crowd_ord[t] = -1; s.crowd_slot[t] = -1; s.tp[t] = 0; s.fp[t] = 0; s.fn[t] = 0; s.iou[t] = acc_iou[t];
  }
  if (tid == 0) { s.n_match = 0; s.n_pred = 0; s.err = 0; }
  __syncthreads();
  const int n = min(*ws.n_pairs, kPqMaxPairs);
  // A: prediction segments (area = all its pixels, VOID intersection), crowd region per category (last in list order)
  for (int i = tid; i < n; i += blockDim.x) {
    const unsigned h = ws.list[i], key = ws.keys[h], c = ws.cnt[h];
    const int ps = pq_pred_slot(s, key & 0xffffu, true);
    if (ps < 0) continue;
    atomicAdd(s.parea + ps, c);
    if ((key >> 16) == kSlotVoid) s.pvoid[ps] = c;
  }
  for (int g = tid; g < G; g += blockDim.x) {
    const long long id = t_id[g], cat = t_cat[g];
    if (id < 1 || id >= (1ll << 24) || (g > 0 && t_id[g - 1] >= id) || cat < 0 || cat >= 255) { atomicOr(&s.err, UPSNET_PQ_E_GT_TABLE); continue; }
    if (t_crowd[g] == 1) atomicMax(s.crowd_ord + cat, (int)t_ord[g]);
  }
  __syncthreads();
  for (int g = tid; g < G; g += blockDim.x) {
    const long long cat = t_cat[g];
    if (t_crowd[g] == 1 && cat >= 0 && cat < 255 && s.crowd_ord[cat] == (int)t_ord[g]) s.crowd_slot[cat] = g;
  }
  __syncthreads();
  // B: matching (:560-579) and the crowd intersection of each prediction segment (:600-601)
  for (int i = tid; i < n; i += blockDim.x) {
    const unsigned h = ws.list[i], key = ws.keys[h], c = ws.cnt[h];
    const int g = (int)(key >> 16);
    if (g >= G) continue;
    const int ps = pq_pred_slot(s, key & 0xffffu, false);
    if (ps < 0) continue;
    const int cls = (int)((key >> 8) & 0xffu);
    if (s.crowd_slot[cls] == g) s.pcrowd[ps] = c;
    if (t_crowd[g] == 1 || t_cat[g] != cls) continue;
    const long long uni = (long long)s.parea[ps] + t_area[g] - (long long)c - (long long)s.pvoid[ps];
    const double iou = (double)c / (double)uni;
    if (iou > 0.5) {
      const int m = atomicAdd(&s.n_match, 1);
      if (m < kPqMaxGt) { s.mkey[m] = key; s.miou[m] = iou; }
      else atomicOr(&s.err, UPSNET_PQ_E_MATCHES);
      s.gmatched[g] = 1;
      s.pmatched[ps] = 1;
    }
  }
  __syncthreads();
  const int nm = min(s.n_match, kPqMaxGt);
  // C: FN (:583-591), FP (:594-606), TP, and the rank of every match
  for (int g = tid; g < G; g += blockDim.x) {
    const long long cat = t_cat[g];
    if (cat >= 0 && cat < 255 && t_crowd[g] != 1 && !s.gmatched[g]) atomicAdd(s.fn + cat, 1);
  }
  for (int ps = tid; ps < kPqPred; ps += blockDim.x) {
    if (s.pkey[ps] == kPqEmpty || s.pmatched[ps]) continue;
    const double frac = (double)(s.pvoid[ps] + s.pcrowd[ps]) / (double)s.parea[ps];
    if (frac > 0.5) continue;
    atomicAdd(s.fp + (s.pkey[ps] >> 8), 1);
  }
  for (int m = tid; m < nm; m += blockDim.x) {
    const unsigned k = s.mkey[m];
    int r = 0;
    for (int q = 0; q < nm; ++q) r += s.mkey[q] < k;
    s.perm[r] = (unsigned short)m;
    atomicAdd(s.tp + ((k >> 8) & 0xffu), 1);
  }
  __syncthreads();
  if (tid == 0)
    for (int r = 0; r < nm; ++r) {
      const int m = s.perm[r];
      s.iou[(s.mkey[m] >> 8) & 0xffu] += s.miou[m];
    }
  __syncthreads();
  for (int t = tid; t < 256; t += blockDim.x) {
    acc_iou[t] = s.iou[t];
    acc[t] += s.tp[t];
    acc[256 + t] += s.fp[t];
    acc[512 + t] += s.fn[t];
  }
  if (tid == 0 && s.err) atomicOr(err, s.err);
  if (tid == 0 && *ws.n_pairs > kPqMaxPairs) atomicOr(err, UPSNET_PQ_E_PAIRS);
}

}  // namespace ups

extern "C" int upsnet_pq_workspace_bytes(size_t* bytes) {
  if (!bytes) return UPSNET_E_BADARG;
  *bytes = ups::pq_ws_layout(nullptr, nullptr);
  return 0;
}

extern "C" int upsnet_pq_update(const unsigned char* pan_2ch, const unsigned char* gt_rgb, int H, int W, const long long* gt_table,
                                int num_gt, const unsigned char* cat_flags, long long* acc_counts, double* acc_iou, int* err,
                                void* workspace, size_t workspace_bytes, void* stream) {
  using namespace ups;
  if (!pan_2ch || !gt_rgb || !cat_flags || !acc_counts || !acc_iou || !err || !workspace || (!gt_table && num_gt > 0))
    return UPSNET_E_BADARG;
  if (H <= 0 || W <= 0 || num_gt < 0) return UPSNET_E_BADARG;
  PqWs ws;
  if (workspace_bytes < pq_ws_layout(&ws, (char*)workspace)) return UPSNET_E_WORKSPACE;
  static bool attr_set[64] = {};                  // the shared-memory opt-in is per device
  int dev = 0;
  UPS_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) return UPSNET_E_UNSUPPORTED;
  if (!attr_set[dev]) {
    UPS_CUDA(cudaFuncSetAttribute(pq_finalize_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(PqFinSmem)));
    attr_set[dev] = true;
  }
  cudaStream_t st = (cudaStream_t)stream;
  UPS_CUDA(cudaMemsetAsync(ws.keys, 0xff, sizeof(unsigned) * kPqHash, st));
  UPS_CUDA(cudaMemsetAsync(ws.cnt, 0, (char*)ws.list - (char*)ws.cnt, st));       // counts and n_pairs
  const size_t HW = (size_t)H * W, nq = (HW + 3) / 4;
  size_t blocks = (nq + 255) / 256;
  if (blocks > (size_t)num_sms() * 6) blocks = (size_t)num_sms() * 6;
  pq_pixel_kernel<<<(unsigned)blocks, 256, 0, st>>>(pan_2ch, gt_rgb, HW, gt_table, num_gt, cat_flags, ws, err);
  UPS_CHECK_LAUNCH();
  pq_finalize_kernel<<<1, kPqFinThreads, sizeof(PqFinSmem), st>>>(gt_table, num_gt, ws, acc_counts, acc_iou, err);
  UPS_CHECK_LAUNCH();
  return 0;
}
