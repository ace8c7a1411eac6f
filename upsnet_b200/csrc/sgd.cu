// sgd.cu -- the optimiser step of the training configuration: the reference's momentum SGD (lib/nn/optimizer.py:80-104)
// with the momentum decay of its training loop (upsnet_end2end_train.py:235-240), over every parameter in one launch.
// See include/upsnet_b200.h for the contract of every symbol.
//
// Multi-tensor and element-wise: one CTA per entry of a caller-owned chunk table, every element owned by one thread,
// no atomics, so the same inputs give the same bytes.  Each reference op is one rounding here, written with explicit
// _rn intrinsics so that nvcc cannot contract b * m into the multiply-add that follows it (torch rounds buf.mul_ on its
// own).  16-byte accesses where the chunk's addresses allow them, scalar ones otherwise; the gradient of a bf16 bucket
// segment may start at any element.
#include "common.cuh"
#include "pair.cuh"

static_assert(sizeof(upsnet_sgd_chunk) == 40, "upsnet_sgd_chunk layout");
static_assert(sizeof(upsnet_sgd_pack_chunk) == 24, "upsnet_sgd_pack_chunk layout");

namespace ups {
namespace {

constexpr int kSgdThreads = 256;

struct SgdGroups {
  double lr[UPSNET_SGD_MAX_GROUPS];
  float wd[UPSNET_SGD_MAX_GROUPS];
  float mom[UPSNET_SGD_MAX_GROUPS];
};

__device__ __forceinline__ float bf16_at(const uint16_t* g, int i) { return __uint_as_float((uint32_t)g[i] << 16); }

// one element: d = g (+ wd p), b = a d + b m, p -= b (b *= 1/10 on a decay step); without momentum p -= d
__device__ __forceinline__ void sgd_update(float& p, float& b, float d, float a, float wd, float m, bool use_wd,
                                           bool use_m, bool decay) {
  if (use_wd) d = __fmaf_rn(wd, p, d);
  if (use_m) {
    b = __fmaf_rn(a, d, __fmul_rn(b, m));
    p = __fsub_rn(p, b);
    if (decay) b = __fmul_rn(b, 0.1f);
  } else {
    p = __fsub_rn(p, d);
  }
}

__device__ __forceinline__ float grad_at(const upsnet_sgd_chunk& c, int i) {
  return c.kind == UPSNET_SGD_GRAD_BF16 ? __fmul_rn(bf16_at((const uint16_t*)c.grad, i), c.inv_world)
                                        : ((const float*)c.grad)[i];
}

__global__ void __launch_bounds__(kSgdThreads) sgd_apply_kernel(const upsnet_sgd_chunk* __restrict__ chunks,
                                                                SgdGroups grp, double lr,
                                                                const double* __restrict__ lr_table,
                                                                const unsigned char* __restrict__ decay_table,
                                                                const int* __restrict__ iteration, int table_begin,
                                                                int table_len) {
  const upsnet_sgd_chunk c = chunks[blockIdx.x];
  bool decay = false;
  if (lr_table) {
    const int k = *iteration - table_begin;
    if (k < 0 || k >= table_len) return;
    lr = lr_table[k];
    decay = decay_table[k] != 0;
  }
  float* __restrict__ p = c.param;
  float* __restrict__ b = c.buf;
  const float m = grp.mom[c.group];
  const bool use_m = m != 0.f;
  if (c.kind == UPSNET_SGD_GRAD_NONE) {  // a buffer without a gradient this step: only the decay touches it
    if (!decay || !use_m) return;
    for (int i = threadIdx.x; i < c.n; i += kSgdThreads) b[i] = __fmul_rn(b[i], 0.1f);
    return;
  }
  const float a = (float)(grp.lr[c.group] * lr);
  const float wd = grp.wd[c.group];
  const bool use_wd = wd != 0.f;
  const bool bf = c.kind == UPSNET_SGD_GRAD_BF16;
  const uintptr_t pb = (uintptr_t)p | (use_m ? (uintptr_t)b : 0);
  const int nq = (pb & 15) ? 0 : c.n >> 2;
  const bool gvec = ((uintptr_t)c.grad & (bf ? 7 : 15)) == 0;
  for (int q = threadIdx.x; q < nq; q += kSgdThreads) {
    float4 pv = reinterpret_cast<const float4*>(p)[q];
    float4 bv = use_m ? reinterpret_cast<const float4*>(b)[q] : make_float4(0.f, 0.f, 0.f, 0.f);
    float d[4];
    if (gvec && bf) {
      const uint2 w = reinterpret_cast<const uint2*>(c.grad)[q];
      d[0] = __fmul_rn(bf16x2_x(w.x), c.inv_world); d[1] = __fmul_rn(bf16x2_y(w.x), c.inv_world);
      d[2] = __fmul_rn(bf16x2_x(w.y), c.inv_world); d[3] = __fmul_rn(bf16x2_y(w.y), c.inv_world);
    } else if (gvec) {
      const float4 g = reinterpret_cast<const float4*>(c.grad)[q];
      d[0] = g.x; d[1] = g.y; d[2] = g.z; d[3] = g.w;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) d[j] = grad_at(c, 4 * q + j);
    }
    sgd_update(pv.x, bv.x, d[0], a, wd, m, use_wd, use_m, decay);
    sgd_update(pv.y, bv.y, d[1], a, wd, m, use_wd, use_m, decay);
    sgd_update(pv.z, bv.z, d[2], a, wd, m, use_wd, use_m, decay);
    sgd_update(pv.w, bv.w, d[3], a, wd, m, use_wd, use_m, decay);
    reinterpret_cast<float4*>(p)[q] = pv;
    if (use_m) reinterpret_cast<float4*>(b)[q] = bv;
  }
  for (int i = 4 * nq + threadIdx.x; i < c.n; i += kSgdThreads) {
    float pv = p[i], bv = use_m ? b[i] : 0.f;
    sgd_update(pv, bv, grad_at(c, i), a, wd, m, use_wd, use_m, decay);
    p[i] = pv;
    if (use_m) b[i] = bv;
  }
}

__device__ __forceinline__ uint16_t bf16_rn(float v) { return __bfloat16_as_ushort(__float2bfloat16_rn(v)); }

__global__ void __launch_bounds__(kSgdThreads) sgd_pack_kernel(const upsnet_sgd_pack_chunk* __restrict__ chunks) {
  const upsnet_sgd_pack_chunk c = chunks[blockIdx.x];
  const float* __restrict__ g = c.grad;
  uint16_t* __restrict__ o = (uint16_t*)c.out;
  const int nq = (((uintptr_t)g & 15) | ((uintptr_t)o & 7)) ? 0 : c.n >> 2;
  for (int q = threadIdx.x; q < nq; q += kSgdThreads) {
    const float4 v = g ? reinterpret_cast<const float4*>(g)[q] : make_float4(0.f, 0.f, 0.f, 0.f);
    reinterpret_cast<uint2*>(o)[q] = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
  }
  for (int i = 4 * nq + threadIdx.x; i < c.n; i += kSgdThreads) o[i] = bf16_rn(g ? g[i] : 0.f);
}

__global__ void sgd_advance_kernel(int* iteration) { *iteration += 1; }

}  // namespace
}  // namespace ups

extern "C" int upsnet_sgd_apply(const upsnet_sgd_chunk* chunks, int num_chunks, int num_groups, const double* group_lr,
                                const float* group_weight_decay, const float* group_momentum, double lr,
                                const double* lr_table, const unsigned char* decay_table, const int* iteration,
                                int table_begin, int table_len, void* stream) {
  using namespace ups;
  if (num_chunks < 0 || num_groups <= 0 || !group_lr || !group_weight_decay || !group_momentum) return UPSNET_E_BADARG;
  if (num_chunks > 0 && !chunks) return UPSNET_E_BADARG;
  if (lr_table && (!decay_table || !iteration || table_len <= 0)) return UPSNET_E_BADARG;
  if (num_groups > UPSNET_SGD_MAX_GROUPS) return UPSNET_E_UNSUPPORTED;
  if (num_chunks == 0) return 0;
  SgdGroups grp{};
  for (int g = 0; g < num_groups; ++g) {
    grp.lr[g] = group_lr[g];
    grp.wd[g] = group_weight_decay[g];
    grp.mom[g] = group_momentum[g];
  }
  sgd_apply_kernel<<<num_chunks, kSgdThreads, 0, (cudaStream_t)stream>>>(chunks, grp, lr, lr_table, decay_table,
                                                                         iteration, table_begin, table_len);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_sgd_pack(const upsnet_sgd_pack_chunk* chunks, int num_chunks, void* stream) {
  using namespace ups;
  if (num_chunks < 0 || (num_chunks > 0 && !chunks)) return UPSNET_E_BADARG;
  if (num_chunks == 0) return 0;
  sgd_pack_kernel<<<num_chunks, kSgdThreads, 0, (cudaStream_t)stream>>>(chunks);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_sgd_advance(int* iteration, void* stream) {
  using namespace ups;
  if (!iteration) return UPSNET_E_BADARG;
  sgd_advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(iteration);
  UPS_CHECK_LAUNCH();
  return 0;
}
