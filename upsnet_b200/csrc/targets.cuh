// targets.cuh -- arithmetic shared by the training-target kernels (rpn_target.cu, proposal_target.cu): bbox.pyx's IoU,
// the seeded draw keys that replace np.random.choice and bbox_transform_inv
#pragma once
#include <cuda_runtime.h>

namespace ups {

__device__ __forceinline__ unsigned long long splitmix64(unsigned long long x) {
  unsigned long long z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// key of candidate position pos in a draw: splitmix64(s ^ pos * golden gamma), s = seed (stream 0) or splitmix64(seed)
// (stream 1); a draw of `size` takes the positions with the `size` smallest keys
__device__ __forceinline__ unsigned long long draw_key(unsigned long long seed, int stream, unsigned long long pos) {
  const unsigned long long s = stream ? splitmix64(seed) : seed;
  return splitmix64(s ^ (pos * 0x9E3779B97F4A7C15ull));
}

// (f64(f32(x2 - x1)) + 1.0) * (f64(f32(y2 - y1)) + 1.0): bbox.pyx's box area as Cython compiles it (the `+ 1` is a
// double literal)
__device__ __forceinline__ double area64(float4 b) {
  return __dmul_rn(__dadd_rn((double)__fsub_rn(b.z, b.x), 1.0), __dadd_rn((double)__fsub_rn(b.w, b.y), 1.0));
}

// bbox.pyx bbox_overlaps for one (box, query box) pair, bit-exact to the compiled extension.  iw and ih are
// f32(f64(f32(min - max)) + 1.0) there; that double rounding is innocuous for a sum of two float32 values (53 >= 2*24 + 1
// bits), so they are the float32 sum computed here.
__device__ __forceinline__ float pair_iou(float4 a, double a_area, float4 q, float q_area) {
  const float iw = __fadd_rn(__fsub_rn(fminf(a.z, q.z), fmaxf(a.x, q.x)), 1.0f);
  if (!(iw > 0.f)) return 0.f;
  const float ih = __fadd_rn(__fsub_rn(fminf(a.w, q.w), fmaxf(a.y, q.y)), 1.0f);
  if (!(ih > 0.f)) return 0.f;
  const float inter = __fmul_rn(iw, ih);
  const float ua = (float)__dsub_rn(__dadd_rn(a_area, (double)q_area), (double)inter);
  return __fdiv_rn(inter, ua);
}

// bbox_transform.py:332-363 bbox_transform_inv, float32: wx * (gt_ctr - ex_ctr) / ex_w (the weight multiplies first),
// ww * log(gt_w / ex_w).  With weights 1 the products are exact, so the RPN targets are those of the unweighted form.
__device__ __forceinline__ float4 box_target(float4 e, float4 g, float4 w) {
  const float ew = __fadd_rn(__fsub_rn(e.z, e.x), 1.0f), eh = __fadd_rn(__fsub_rn(e.w, e.y), 1.0f);
  const float ecx = __fadd_rn(e.x, __fmul_rn(0.5f, ew)), ecy = __fadd_rn(e.y, __fmul_rn(0.5f, eh));
  const float gw = __fadd_rn(__fsub_rn(g.z, g.x), 1.0f), gh = __fadd_rn(__fsub_rn(g.w, g.y), 1.0f);
  const float gcx = __fadd_rn(g.x, __fmul_rn(0.5f, gw)), gcy = __fadd_rn(g.y, __fmul_rn(0.5f, gh));
  return make_float4(__fdiv_rn(__fmul_rn(w.x, __fsub_rn(gcx, ecx)), ew),
                     __fdiv_rn(__fmul_rn(w.y, __fsub_rn(gcy, ecy)), eh), __fmul_rn(w.z, logf(__fdiv_rn(gw, ew))),
                     __fmul_rn(w.w, logf(__fdiv_rn(gh, eh))));
}

}  // namespace ups
