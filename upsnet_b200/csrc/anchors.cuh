// anchors.cuh -- the shifted anchor of one feature cell, shared by the RPN decode (detection.cu) and the RPN training
// targets (rpn_target.cu)
#pragma once
#include <cuda_runtime.h>

namespace ups {

// float32(cell anchor (float64) + shift): the shifted anchors of pyramid_proposal.py:83-100 / bbox_transform.py:298 and
// the field of anchors of generate_anchors.py:79-130 are both added in float64 and cast to float32 afterwards
__device__ __forceinline__ float4 shifted_anchor(const double* cell, int x, int y, int stride) {
  const double sx = (double)(x * stride), sy = (double)(y * stride);
  return make_float4((float)(cell[0] + sx), (float)(cell[1] + sy), (float)(cell[2] + sx), (float)(cell[3] + sy));
}

}  // namespace ups
