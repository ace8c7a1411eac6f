// pair.cuh -- the bf16x2 word and the hi/lo bf16 pair format, written down once.
//
// A hi/lo pair (UPSNET_DTYPE_PAIR in include/upsnet_b200.h, operators.Pair in Python) stores an fp32 value v as
// hi = bf16(v) and lo = bf16(v - hi); hi + lo is exact in fp32.  A pair tensor is NHWC with 2C bf16 channels per pixel,
// [0,C) the hi values and [C,2C) the lo values.  Kernels move bf16 in 32-bit words of two elements: element x (the
// lower address) is the low half, so as fp32 it is `w << 16`, and element y is `w & 0xffff0000`.
// Every kernel packs, unpacks, splits and blends this format through the functions below; each keeps the evaluation
// order of the expressions it replaced, so results are bit-identical to the inline forms.
#pragma once
#include <cuda_bf16.h>
#include <cstdint>

namespace ups {

// ---- one bf16x2 word ----
__device__ __forceinline__ float bf16x2_x(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf16x2_y(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
// both elements as a packed fp32 pair (low word = element x), the operand form of f32x2_fma / f32x2_add
__device__ __forceinline__ unsigned long long bf16x2_to_f32x2(uint32_t w) {
  unsigned long long r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "r"(w << 16), "r"(w & 0xffff0000u));
  return r;
}

// packed fp32 pairs (low word = first value): element-wise fma / add
__device__ __forceinline__ unsigned long long f32x2_fma(unsigned long long a, unsigned long long b, unsigned long long c) {
  const float r0 = fmaf(__uint_as_float((uint32_t)a), __uint_as_float((uint32_t)b), __uint_as_float((uint32_t)c));
  const float r1 = fmaf(__uint_as_float((uint32_t)(a >> 32)), __uint_as_float((uint32_t)(b >> 32)), __uint_as_float((uint32_t)(c >> 32)));
  return ((unsigned long long)__float_as_uint(r1) << 32) | __float_as_uint(r0);
}
__device__ __forceinline__ unsigned long long f32x2_add(unsigned long long a, unsigned long long b) {
  const float r0 = __uint_as_float((uint32_t)a) + __uint_as_float((uint32_t)b);
  const float r1 = __uint_as_float((uint32_t)(a >> 32)) + __uint_as_float((uint32_t)(b >> 32));
  return ((unsigned long long)__float_as_uint(r1) << 32) | __float_as_uint(r0);
}

// ---- hi/lo pairs ----
// the value of element x / y of a pair, from its hi word h and lo word l (exact)
__device__ __forceinline__ float pair_x(uint32_t h, uint32_t l) { return bf16x2_x(h) + bf16x2_x(l); }
__device__ __forceinline__ float pair_y(uint32_t h, uint32_t l) { return bf16x2_y(h) + bf16x2_y(l); }
// the lo word bf16(a - hi), bf16(b - hi) that goes with the hi word hi = pack_bf16x2(a, b)
__device__ __forceinline__ uint32_t pair_lo2(float a, float b, uint32_t hi) {
  return pack_bf16x2(a - bf16x2_x(hi), b - bf16x2_y(hi));
}
// (a, b) -> hi word bf16(a), bf16(b) and its lo word
__device__ __forceinline__ void split_pair2(float a, float b, uint32_t& hi, uint32_t& lo) {
  hi = pack_bf16x2(a, b);
  lo = pair_lo2(a, b, hi);
}
// the same for eight consecutive values and 16-byte vectors
__device__ __forceinline__ uint4 pack_bf16x8(const float* o) {
  return make_uint4(pack_bf16x2(o[0], o[1]), pack_bf16x2(o[2], o[3]), pack_bf16x2(o[4], o[5]), pack_bf16x2(o[6], o[7]));
}
__device__ __forceinline__ uint4 pair_lo8(const float* o, const uint4& hi) {
  return make_uint4(pair_lo2(o[0], o[1], hi.x), pair_lo2(o[2], o[3], hi.y), pair_lo2(o[4], o[5], hi.z), pair_lo2(o[6], o[7], hi.w));
}
__device__ __forceinline__ void split_pair8(const float* o, uint4& hi, uint4& lo) {
  split_pair2(o[0], o[1], hi.x, lo.x);
  split_pair2(o[2], o[3], hi.y, lo.y);
  split_pair2(o[4], o[5], hi.z, lo.z);
  split_pair2(o[6], o[7], hi.w, lo.w);
}
// one value -> its hi and lo bf16 (the weight packs)
__device__ __forceinline__ void split_bf16(float v, __nv_bfloat16& h, __nv_bfloat16& l) {
  h = __float2bfloat16_rn(v);
  l = __float2bfloat16_rn(v - __bfloat162float(h));
}

// Bilinear blend of 8 channels of a pair tensor, split again: corner i has weight w[i] (x, y, z, w) and the 16-byte hi / lo
// vectors hc[i] / lc[i].  The deformable gathers are issue-bound, so it is written for instruction count: the hi plane is
// blended with fp32 FMAs on channel pairs (exact products of the bf16 values), the lo plane in packed bf16x2 HFMA2 with
// bf16-rounded weights (the lo plane is 2^-9 of the value, its blend needs 2^-9 relative accuracy only, 2^-18 overall),
// and the two sums are added in fp32.
__device__ __forceinline__ void pair_blend8(const float4& w, const uint4 (&hc)[4], const uint4 (&lc)[4], uint4& hi, uint4& lo) {
  const float wf[4] = {w.x, w.y, w.z, w.w};
  unsigned long long acc[4] = {0ull, 0ull, 0ull, 0ull};      // fp32x2: channels (2q, 2q + 1)
  __nv_bfloat162 lacc[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t hw[4] = {hc[i].x, hc[i].y, hc[i].z, hc[i].w};
    const uint32_t lw[4] = {lc[i].x, lc[i].y, lc[i].z, lc[i].w};
    const __nv_bfloat162 wb = __float2bfloat162_rn(wf[i]);
    unsigned long long wp;
    asm("mov.b64 %0, {%1, %1};" : "=l"(wp) : "r"(__float_as_uint(wf[i])));
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      acc[q] = f32x2_fma(wp, bf16x2_to_f32x2(hw[q]), acc[q]);
      const __nv_bfloat162 lv = *reinterpret_cast<const __nv_bfloat162*>(&lw[q]);
      lacc[q] = i == 0 ? __hmul2(wb, lv) : __hfma2(wb, lv, lacc[q]);
    }
  }
  uint32_t h[4], l[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    acc[q] = f32x2_add(acc[q], bf16x2_to_f32x2(*reinterpret_cast<const uint32_t*>(&lacc[q])));
    uint32_t a0, a1;
    asm("mov.b64 {%0, %1}, %2;" : "=r"(a0), "=r"(a1) : "l"(acc[q]));
    split_pair2(__uint_as_float(a0), __uint_as_float(a1), h[q], l[q]);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}

}  // namespace ups
