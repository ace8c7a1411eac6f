// cta.cuh -- CTA-wide building blocks of the data kernels (detection glue, training targets, evaluators, losses): the
// order-preserving float key, exclusive scan, ordered compaction by ballot rank, radix select of the k-th key, bitonic
// sort in shared memory and fixed-order partial sums.  A routine with a Threads parameter is called by all Threads
// threads of the CTA.
#pragma once
#include <cuda_runtime.h>

namespace ups {

// float -> unsigned whose unsigned order is the float order (-0 just below +0, NaNs beyond the infinities), and back
__device__ __forceinline__ unsigned orderable(float f) {
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float from_orderable(unsigned o) {
  return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

// Exclusive sum of one value per thread in thread order, and in *total the sum over the CTA (every thread).  warp_sums is
// Threads / 32 values of shared memory, free again on return.  Hand-written rather than cub::BlockScan: at 1024 threads
// (ptxas, sm_90a) CUB's raking scan took pt_sample_kernel from 32 to 60 registers, rt_scan_kernel from 32 to 57, and
// pan_prep_kernel from 32 to 64 with 144 bytes of spill stores.
template <int Threads, typename T>
__device__ __forceinline__ T cta_scan_excl(T v, T* warp_sums, T* total) {
  constexpr int kWarps = Threads / 32;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  T x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[wid] = x;
  __syncthreads();
  if (wid == 0) {
    T w = lane < kWarps ? warp_sums[lane] : T(0);
#pragma unroll
    for (int o = 1; o < kWarps; o <<= 1) {
      const T y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    if (lane < kWarps) warp_sums[lane] = w;   // inclusive
  }
  __syncthreads();
  const T base = wid ? warp_sums[wid - 1] : T(0);
  *total = warp_sums[kWarps - 1];
  __syncthreads();
  return base + x - v;
}

// Ordered compaction: the number of threads below this one (in thread order) whose flag is set, and in *total the
// number of set flags.  warp_n is Threads / 32 ints of shared memory, free again on return.
template <int Threads>
__device__ __forceinline__ int cta_ballot_rank(bool flag, int* warp_n, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned bal = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) warp_n[warp] = __popc(bal);
  __syncthreads();
  int rank = __popc(bal & ((1u << lane) - 1u)), n = 0;
  for (int w = 0; w < Threads / 32; ++w) {
    if (w < warp) rank += warp_n[w];
    n += warp_n[w];
  }
  __syncthreads();
  *total = n;
  return rank;
}

struct RadixDigit {
  int digit;   // the bin that holds the need-th key
  int need;    // how many keys of that bin are still to be taken, >= 1
};

// One digit of a radix select, by one full warp: hist holds the Bins counts of the keys whose higher digits are fixed,
// and the need-th key (1 <= need <= the sum of hist) in scan order, from the top bin down when Largest, is found.  Lane l
// owns scan positions [l * Bins / 32, (l + 1) * Bins / 32).  Returns true in the one lane that owns the digit, which
// writes the result; *r is set in that lane only.
template <int Bins, bool Largest>
__device__ __forceinline__ bool warp_radix_digit(const unsigned* hist, int need, RadixDigit* r) {
  constexpr int kPer = Bins / 32;
  static_assert(kPer * 32 == Bins, "whole bins per lane");
  const int lane = threadIdx.x & 31;
  auto bin = [&](int j) { const int b = lane * kPer + j; return Largest ? Bins - 1 - b : b; };
  unsigned mine = 0;
  for (int j = 0; j < kPer; ++j) mine += hist[bin(j)];
  unsigned incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane != __ffs(__ballot_sync(0xffffffffu, incl >= (unsigned)need)) - 1) return false;
  unsigned acc = incl - mine;
  int j = 0;
  for (; j < kPer - 1 && acc + hist[bin(j)] < (unsigned)need; ++j) acc += hist[bin(j)];
  r->digit = bin(j);
  r->need = need - (int)acc;
  return true;
}

// The k-th largest (Largest) or k-th smallest of the n keys key_at(0), ..., key_at(n - 1), 1 <= k <= n: an exact radix
// select over the low KeyBits bits of Key, DigitBits per pass from the top, each pass a shared-memory histogram.
template <int Threads, typename Key, int KeyBits, int DigitBits, bool Largest, class KeyAt>
__device__ Key cta_radix_select(const KeyAt& key_at, int n, int k) {
  constexpr int kBins = 1 << DigitBits, kPasses = (KeyBits + DigitBits - 1) / DigitBits;
  __shared__ unsigned hist[kBins];
  __shared__ Key s_prefix;
  __shared__ int s_need;
  for (int pass = 0; pass < kPasses; ++pass) {
    const int shift = (kPasses - 1 - pass) * DigitBits;
    const Key mask_hi = pass == 0 ? Key(0) : ~Key(0) << (shift + DigitBits);
    for (int b = threadIdx.x; b < kBins; b += Threads) hist[b] = 0u;
    __syncthreads();
    const Key prefix = pass == 0 ? Key(0) : s_prefix;
    for (int i = threadIdx.x; i < n; i += Threads) {
      const Key key = key_at(i);
      if ((key & mask_hi) == prefix) atomicAdd(&hist[(unsigned)(key >> shift) & (kBins - 1)], 1u);
    }
    __syncthreads();
    RadixDigit d;
    if (threadIdx.x < 32 && warp_radix_digit<kBins, Largest>(hist, pass == 0 ? k : s_need, &d)) {
      s_prefix = prefix | ((Key)d.digit << shift);
      s_need = d.need;
    }
    __syncthreads();
  }
  return s_prefix;
}

// The fence-and-ticket step of a pass split over nblocks CTAs: true, in every thread, in the CTA that takes the last
// ticket, which then sees every global write the other CTAs made before taking theirs.  The caller re-arms *ticket.
__device__ __forceinline__ bool last_cta(unsigned* ticket, unsigned nblocks) {
  __shared__ bool s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(ticket, 1u) == nblocks - 1;
  __syncthreads();
  if (!s_last) return false;
  __threadfence();
  return true;
}

// Sorts keys[0, n) in shared memory, n a power of two >= 2; the keys are in place when it returns.
template <int Threads, bool Descending, typename Key>
__device__ __forceinline__ void cta_bitonic_sort(Key* keys, int n) {
  for (int k = 2; k <= n; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < n / 2; t += Threads) {
        const int lo = ((t / j) * (j << 1)) + (t % j), hi = lo + j;
        const Key a = keys[lo], b = keys[hi];
        const bool first = (lo & k) == 0;      // this pair is ordered in the direction of the whole sort
        if ((Descending ? a < b : a > b) == first) { keys[lo] = b; keys[hi] = a; }
      }
      __syncthreads();
    }
}

// Per-block sums of ND doubles and NI ints in a fixed order (lanes by shuffle, warps by thread 0), written to slot
// blockIdx.x of pd [nblocks, ND] and pi [nblocks, NI].
template <int Threads, int ND, int NI>
__device__ __forceinline__ void cta_partials(double (&d)[ND], int (&n)[NI], double* pd, int* pi) {
  __shared__ double s_d[Threads / 32][ND];
  __shared__ int s_i[Threads / 32][NI];
  for (int o = 16; o; o >>= 1) {
#pragma unroll
    for (int j = 0; j < ND; ++j) d[j] += __shfl_down_sync(0xffffffffu, d[j], o);
#pragma unroll
    for (int j = 0; j < NI; ++j) n[j] += __shfl_down_sync(0xffffffffu, n[j], o);
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) {
#pragma unroll
    for (int j = 0; j < ND; ++j) s_d[wid][j] = d[j];
#pragma unroll
    for (int j = 0; j < NI; ++j) s_i[wid][j] = n[j];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < Threads / 32; ++k) {
#pragma unroll
      for (int j = 0; j < ND; ++j) d[j] += s_d[k][j];
#pragma unroll
      for (int j = 0; j < NI; ++j) n[j] += s_i[k][j];
    }
#pragma unroll
    for (int j = 0; j < ND; ++j) pd[(size_t)blockIdx.x * ND + j] = d[j];
#pragma unroll
    for (int j = 0; j < NI; ++j) pi[(size_t)blockIdx.x * NI + j] = n[j];
  }
}

// Second stage, one CTA: the sums of all nblocks partials of cta_partials in a fixed order (strided per thread, then a
// tree); valid in every thread on return.
template <int Threads, int ND, int NI>
__device__ __forceinline__ void cta_sum_partials(const double* pd, const int* pi, int nblocks, double (&d)[ND],
                                                 int (&n)[NI]) {
  __shared__ double s_d[Threads][ND];
  __shared__ int s_i[Threads][NI];
  const int t = threadIdx.x;
#pragma unroll
  for (int j = 0; j < ND; ++j) s_d[t][j] = 0.0;
#pragma unroll
  for (int j = 0; j < NI; ++j) s_i[t][j] = 0;
  for (int b = t; b < nblocks; b += Threads) {
#pragma unroll
    for (int j = 0; j < ND; ++j) s_d[t][j] += pd[(size_t)b * ND + j];
#pragma unroll
    for (int j = 0; j < NI; ++j) s_i[t][j] += pi[(size_t)b * NI + j];
  }
  __syncthreads();
  for (int o = Threads / 2; o; o >>= 1) {
    if (t < o) {
#pragma unroll
      for (int j = 0; j < ND; ++j) s_d[t][j] += s_d[t + o][j];
#pragma unroll
      for (int j = 0; j < NI; ++j) s_i[t][j] += s_i[t + o][j];
    }
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < ND; ++j) d[j] = s_d[0][j];
#pragma unroll
  for (int j = 0; j < NI; ++j) n[j] = s_i[0][j];
}

}  // namespace ups
