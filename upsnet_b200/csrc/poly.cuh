// poly.cuh -- the edge walk of cocoapi maskApi.c rleFrPoly on an h x w canvas, shared by the 28x28 mask targets
// (proposal_target.cu, h = w = M) and the ground-truth rasteriser of the COCO evaluation (gt_rle.cu, the image's h x w).
//
// rleFrPoly walks each edge at 5x, keeps the points where the upsampled x coordinate u changes and min(u) = 5n + 2 (a
// pixel centre, 0 <= n < w), maps each to (x = n, y = ceil(clamp((min v + .5) / 5 - .5, 0, h))), sorts the column-major
// indices a = x * h + y, differences them and merges zero runs.  The runs alternate 0 / 1 starting with 0, so pixel i is
// 1 iff an odd number of points have a <= i: a zero difference (two equal points) cancels a boundary, which is what the
// merge does.  So each surviving point toggles index a and a prefix XOR gives the mask.  A point with y = h toggles
// a = (n + 1) * h, row 0 of the next column, exactly where maskApi.c's sorted index puts it; a = h * w (the last
// column) falls off the end.  Within an edge u moves by at most 1 per point, monotonically, so each n is crossed at most
// once: on a shallow edge u = t + xs and the crossing is direct; on a steep edge u(t) = (int)(xs + s*t + .5) and the
// crossing is found by bisection on that same double expression.  Consecutive edges share the rounded vertex when it is
// >= 0; when it is negative, (int) truncation can make them differ, but then both u <= 0 and the pair is dropped by
// xd < 0.  Edges are thus independent, and the toggles of one edge are a function of (edge, n) alone, so any number of
// threads can share one edge's columns (tests/proposal_target_oracle.py and tests/gt_rle_oracle.py pin this
// formulation to the literal rleFrPoly).  Every rounding step is an explicit _rn intrinsic: gcc's x86-64 build of
// maskApi.c and numpy do not contract into FMA.
#pragma once
#include <cuda_runtime.h>

namespace ups {

// (int)(5 * c + .5), as rleFrPoly rounds the scaled vertices (double, truncation)
__device__ __forceinline__ int up5(double c) { return (int)__dadd_rn(__dmul_rn(5.0, c), 0.5); }
__device__ __forceinline__ int up5(float c) { return up5((double)c); }

// One edge (X0, Y0) -> (X1, Y1) of rounded vertices, oriented as rleFrPoly walks it, and the columns it crosses.
struct PolyEdge {
  double s;          // dy / dx (shallow) or dx / dy (steep) after the flip
  int xs, ys, dy;    // start after the flip; dy: the steep walk's length
  int n0, n1;        // crossed columns n0..n1 (none when n0 > n1), n1 <= w - 1
  bool steep;
};

__device__ __forceinline__ int poly_u(const PolyEdge& e, int t) {
  return (int)__dadd_rn(__dadd_rn((double)e.xs, __dmul_rn(e.s, (double)t)), 0.5);
}

__device__ __forceinline__ PolyEdge poly_edge(int X0, int Y0, int X1, int Y1, int w) {
  PolyEdge e;
  const int dx = abs(X1 - X0), dy = abs(Y1 - Y0);
  e.steep = dx < dy;
  int lo, hi;
  if (!e.steep) {
    const bool flip = X0 > X1;
    e.xs = flip ? X1 : X0;
    e.ys = flip ? Y1 : Y0;
    const int ye = flip ? Y0 : Y1;
    e.s = dx ? __ddiv_rn((double)(ye - e.ys), (double)dx) : 0.0;    // dx == 0: one point, no column is crossed
    e.dy = 0;
    lo = e.xs;
    hi = e.xs + dx;
  } else {
    const bool flip = Y0 > Y1;
    e.xs = flip ? X1 : X0;
    const int xe = flip ? X0 : X1;
    e.ys = flip ? Y1 : Y0;
    e.s = __ddiv_rn((double)(xe - e.xs), (double)dy);
    e.dy = dy;
    const int u0 = poly_u(e, 0), u1 = poly_u(e, dy);
    lo = min(u0, u1);
    hi = max(u0, u1);
  }
  e.n0 = lo <= 2 ? 0 : (lo - 2 + 4) / 5;
  e.n1 = hi < 3 ? -1 : min(w - 1, (hi - 3) / 5);
  return e;
}

// min(v) of the boundary point where the edge crosses column n (e.n0 <= n <= e.n1), for a shallow or a steep edge
template <bool Steep>
__device__ __forceinline__ int poly_edge_v(const PolyEdge& e, int n) {
  if (!Steep) {
    const int ta = 5 * n + 2 - e.xs;
    const int va = (int)__dadd_rn(__dadd_rn((double)e.ys, __dmul_rn(e.s, (double)ta)), 0.5);
    const int vb = (int)__dadd_rn(__dadd_rn((double)e.ys, __dmul_rn(e.s, (double)(ta + 1))), 0.5);
    return min(va, vb);
  }
  const int xd = 5 * n + 2;
  int a = 0, b = e.dy;              // the first t past the crossing: u(t) >= xd + 1 (s > 0) or u(t) <= xd (s < 0)
  while (b - a > 1) {
    const int m = (a + b) >> 1;
    const int um = poly_u(e, m);
    if (e.s > 0.0 ? um >= xd + 1 : um <= xd) b = m;
    else a = m;
  }
  return e.ys + b - 1;
}

// the row y of a boundary point of min(v) = yv: ceil(clamp((yv + .5) / 5 - .5, 0, h))
__device__ __forceinline__ int poly_row(int yv, int h) {
  double yd = __dsub_rn(__ddiv_rn(__dadd_rn((double)yv, 0.5), 5.0), 0.5);
  if (yd < 0.0) yd = 0.0;
  else if (yd > (double)h) yd = (double)h;
  return (int)ceil(yd);
}

// the toggled column-major index n * h + y of the point on column n; h * w and beyond fall off the canvas
__device__ __forceinline__ int poly_toggle_index(const PolyEdge& e, int n, int h) {
  return n * h + poly_row(e.steep ? poly_edge_v<true>(e, n) : poly_edge_v<false>(e, n), h);
}

// Every toggle of one edge into a bitmap of h * w bits (one thread walks the edge: at most w steps)
__device__ __forceinline__ void edge_toggles(unsigned int* bits, int h, int w, int X0, int Y0, int X1, int Y1) {
  const PolyEdge e = poly_edge(X0, Y0, X1, Y1, w);
  auto toggle = [&](int yv, int n) {
    const int a = n * h + poly_row(yv, h);
    if (a < h * w) atomicXor(bits + (a >> 5), 1u << (a & 31));
  };
  if (e.steep) for (int n = e.n0; n <= e.n1; ++n) toggle(poly_edge_v<true>(e, n), n);
  else for (int n = e.n0; n <= e.n1; ++n) toggle(poly_edge_v<false>(e, n), n);
}

}  // namespace ups
