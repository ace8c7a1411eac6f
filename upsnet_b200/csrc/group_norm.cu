// group_norm.cu -- GroupNorm (nn.GroupNorm semantics: biased variance, eps inside the root) over the NHWC activations
// of the engine and of the training forward: forward for whole maps and for roi rows, backward for whole maps.
// See include/upsnet_b200.h for the contract of every symbol.
//
// Deterministic: no atomics; every sum and every merge of partial statistics runs in a fixed order, so the same input
// gives the same bytes, also under graph replay.  Partial statistics are (count, mean, M2) triples merged by Chan's
// formula, which keeps the variance of a group of ~10^6 values (P2 at 1024x2048) accurate in fp32.
//
// Map kernels: a CTA of 256 threads covers all C channels of kChunk-pixel chunks; thread t owns channels
// (t % TC) + j TC (TC = min(C, 256), j < C / TC) at pixel offset t / TC of each chunk, so its channels stay fixed and
// a warp reads consecutive channels.
#include <math.h>

#include "common.cuh"
#include "pair.cuh"

namespace ups {
namespace {

constexpr int kGnThreads = 256;
constexpr int kGnChunk = 64;        // pixels per chunk
constexpr int kGnMaxJ = 4;          // C <= 1024
constexpr int kGnMaxBlocks = 512;   // statistics CTAs per image
constexpr int kGnMaxC = 1024;

struct Stat {
  float n, mean, m2;
};

// Chan et al.: the statistics of the union of two disjoint sets
__device__ __forceinline__ Stat chan_merge(Stat a, Stat b) {
  if (b.n == 0.f) return a;
  if (a.n == 0.f) return b;
  const float n = a.n + b.n;
  const float d = b.mean - a.mean;
  const float fb = b.n / n;
  return Stat{n, a.mean + d * fb, a.m2 + b.m2 + d * d * a.n * fb};
}

__device__ __forceinline__ float load_elem(const void* x, int dtype, size_t pix, int C, int c) {
  if (dtype == UPSNET_DTYPE_F32) return static_cast<const float*>(x)[pix * C + c];
  const __nv_bfloat16* b = static_cast<const __nv_bfloat16*>(x);
  if (dtype == UPSNET_DTYPE_BF16) return __bfloat162float(b[pix * C + c]);
  return __bfloat162float(b[pix * 2 * C + c]) + __bfloat162float(b[pix * 2 * C + C + c]);
}

__device__ __forceinline__ void store_elem(void* y, int dtype, size_t pix, int C, int c, float v) {
  if (dtype == UPSNET_DTYPE_F32) {
    static_cast<float*>(y)[pix * C + c] = v;
    return;
  }
  __nv_bfloat16* b = static_cast<__nv_bfloat16*>(y);
  if (dtype == UPSNET_DTYPE_BF16) {
    b[pix * C + c] = __float2bfloat16_rn(v);
    return;
  }
  __nv_bfloat16 h, l;
  split_bf16(v, h, l);
  b[pix * 2 * C + c] = h;
  b[pix * 2 * C + C + c] = l;
}

struct MapGeom {
  int C, HW, W, groups, TC, SUB, J, nchunks;
};

__host__ __device__ inline MapGeom map_geom(int C, int H, int W, int groups) {
  MapGeom g;
  g.C = C;
  g.HW = H * W;
  g.W = W;
  g.groups = groups;
  g.TC = C < kGnThreads ? C : kGnThreads;
  g.SUB = kGnThreads / g.TC;
  g.J = C / g.TC;
  g.nchunks = (g.HW + kGnChunk - 1) / kGnChunk;
  return g;
}

// Phase 1: per (image, group, CTA) partial statistics.  Each thread folds every chunk it visits into its running
// (count, mean, M2) per channel: the chunk's shifted sums (shift = its first value) give the chunk's mean and M2, which
// are merged by Chan's formula.  Then thread `g` merges the group's channels and sub-slots in a fixed order.
__global__ void __launch_bounds__(kGnThreads)
gn_stats_kernel(const void* __restrict__ x, int dtype, MapGeom gm, float* __restrict__ part) {
  __shared__ Stat sh[kGnThreads][kGnMaxJ];
  const int n = blockIdx.y, t = threadIdx.x;
  const int c0 = t % gm.TC, sub = t / gm.TC;
  Stat acc[kGnMaxJ];
#pragma unroll
  for (int j = 0; j < kGnMaxJ; ++j) acc[j] = Stat{0.f, 0.f, 0.f};
  for (int ch = blockIdx.x; ch < gm.nchunks; ch += gridDim.x) {
    const int p0 = ch * kGnChunk;
    const int p1 = min(p0 + kGnChunk, gm.HW);
#pragma unroll
    for (int j = 0; j < kGnMaxJ; ++j) {
      if (j >= gm.J) break;
      const int c = c0 + j * gm.TC;
      float k = 0.f, s1 = 0.f, s2 = 0.f, cnt = 0.f;
      for (int p = p0 + sub; p < p1; p += gm.SUB) {
        const float v = load_elem(x, dtype, (size_t)n * gm.HW + p, gm.C, c);
        if (cnt == 0.f) k = v;
        const float d = v - k;
        s1 += d;
        s2 = fmaf(d, d, s2);
        cnt += 1.f;
      }
      if (cnt > 0.f) {
        const float m = s1 / cnt;
        acc[j] = chan_merge(acc[j], Stat{cnt, k + m, fmaxf(s2 - s1 * m, 0.f)});
      }
    }
  }
#pragma unroll
  for (int j = 0; j < kGnMaxJ; ++j) sh[t][j] = acc[j];
  __syncthreads();
  const int cg = gm.C / gm.groups;
  for (int g = t; g < gm.groups; g += kGnThreads) {
    Stat s{0.f, 0.f, 0.f};
    for (int c = g * cg; c < (g + 1) * cg; ++c)
      for (int u = 0; u < gm.SUB; ++u) s = chan_merge(s, sh[u * gm.TC + c % gm.TC][c / gm.TC]);
    float* o = part + (((size_t)n * gm.groups + g) * gridDim.x + blockIdx.x) * 3;
    o[0] = s.n;
    o[1] = s.mean;
    o[2] = s.m2;
  }
}

// Merge the CTA partials of one (image, group): one warp, lane-strided in order, then a fixed shuffle-down tree.
// stats[(n G + g) 2 + {0, 1}] = mean, 1 / sqrt(var + eps).
__global__ void gn_finalize_kernel(const float* __restrict__ part, int nparts, int total, float eps,
                                   float* __restrict__ stats) {
  const int w = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x % 32;
  if (w >= total) return;
  const float* p = part + (size_t)w * nparts * 3;
  Stat s{0.f, 0.f, 0.f};
  for (int i = lane; i < nparts; i += 32) s = chan_merge(s, Stat{p[3 * i], p[3 * i + 1], p[3 * i + 2]});
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    Stat o{__shfl_down_sync(0xffffffffu, s.n, off), __shfl_down_sync(0xffffffffu, s.mean, off),
           __shfl_down_sync(0xffffffffu, s.m2, off)};
    s = chan_merge(s, o);
  }
  if (lane == 0) {
    stats[2 * w] = s.mean;
    stats[2 * w + 1] = 1.f / sqrtf(s.m2 / s.n + eps);
  }
}

// Phase 2: y = (x - mean) rstd gamma + beta [+ shift[n]] [+ up2(residual)] [ReLU], written in y's format.
__global__ void __launch_bounds__(kGnThreads)
gn_apply_kernel(const void* __restrict__ x, const float* __restrict__ stats, const float* __restrict__ gamma,
                const float* __restrict__ beta, const float* __restrict__ shift, const void* __restrict__ res,
                void* __restrict__ y, int dtype, MapGeom gm, int flags) {
  const int n = blockIdx.y, t = threadIdx.x;
  const int c0 = t % gm.TC, sub = t / gm.TC;
  const int cg = gm.C / gm.groups;
  const bool relu = flags & UPSNET_EPI_RELU, up2 = res != nullptr;
  const int Wr = gm.W / 2, HWr = (gm.HW / gm.W / 2) * Wr;
  float mean[kGnMaxJ], a[kGnMaxJ], b[kGnMaxJ];
#pragma unroll
  for (int j = 0; j < kGnMaxJ; ++j) {
    if (j >= gm.J) break;
    const int c = c0 + j * gm.TC, g = c / cg;
    mean[j] = stats[2 * ((size_t)n * gm.groups + g)];
    a[j] = stats[2 * ((size_t)n * gm.groups + g) + 1] * gamma[c];
    b[j] = beta[c] + (shift ? shift[(size_t)n * gm.C + c] : 0.f);
  }
  for (int ch = blockIdx.x; ch < gm.nchunks; ch += gridDim.x) {
    const int p1 = min(ch * kGnChunk + kGnChunk, gm.HW);
    for (int p = ch * kGnChunk + sub; p < p1; p += gm.SUB) {
      const size_t pix = (size_t)n * gm.HW + p;
      size_t rpix = 0;
      if (up2) rpix = (size_t)n * HWr + (size_t)(p / gm.W / 2) * Wr + (p % gm.W) / 2;
#pragma unroll
      for (int j = 0; j < kGnMaxJ; ++j) {
        if (j >= gm.J) break;
        const int c = c0 + j * gm.TC;
        float v = (load_elem(x, dtype, pix, gm.C, c) - mean[j]) * a[j] + b[j];
        if (up2) v += load_elem(res, dtype, rpix, gm.C, c);
        if (relu) v = fmaxf(v, 0.f);
        store_elem(y, dtype, pix, gm.C, c, v);
      }
    }
  }
}

// Row GroupNorm: one warp per (row, group) of rows of HW pixels x C channels (NHWC), all in one launch.  Two passes over
// the group (mean, then the sum of squared deviations) in lane order and a fixed shuffle tree, then the apply.
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_down_sync(0xffffffffu, v, off);
  return __shfl_sync(0xffffffffu, v, 0);
}

__global__ void gn_rows_kernel(const void* __restrict__ x, const float* __restrict__ gamma,
                               const float* __restrict__ beta, void* __restrict__ y, int R, int C, int HW,
                               int groups, float eps, int dtype, int flags, const int* __restrict__ n_dev) {
  const int w = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x % 32;
  const int r = w / groups, g = w % groups;
  if (r >= R || (n_dev && r >= *n_dev)) return;
  const int cg = C / groups, M = HW * cg;
  float s = 0.f;
  for (int e = lane; e < M; e += 32) s += load_elem(x, dtype, (size_t)r * HW + e / cg, C, g * cg + e % cg);
  const float mean = warp_sum(s) / (float)M;
  s = 0.f;
  for (int e = lane; e < M; e += 32) {
    const float d = load_elem(x, dtype, (size_t)r * HW + e / cg, C, g * cg + e % cg) - mean;
    s = fmaf(d, d, s);
  }
  const float rstd = 1.f / sqrtf(warp_sum(s) / (float)M + eps);
  for (int e = lane; e < M; e += 32) {
    const int c = g * cg + e % cg;
    const size_t pix = (size_t)r * HW + e / cg;
    float v = (load_elem(x, dtype, pix, C, c) - mean) * (rstd * gamma[c]) + beta[c];
    if (flags & UPSNET_EPI_RELU) v = fmaxf(v, 0.f);
    store_elem(y, dtype, pix, C, c, v);
  }
}

// ---- backward (fp32 NHWC) ----
__device__ __forceinline__ float gn_dz(const float* dy, const float* y, size_t i) {
  const float d = dy[i];
  return (y && !(y[i] > 0.f)) ? 0.f : d;
}

// per (image, CTA, channel): sum dz and sum dz * xhat over the CTA's chunks, sub-slots merged in order
__global__ void __launch_bounds__(kGnThreads)
gn_bwd_reduce_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ y,
                     const float* __restrict__ stats, MapGeom gm, float* __restrict__ part) {
  __shared__ float sh[kGnThreads][kGnMaxJ][2];
  const int n = blockIdx.y, t = threadIdx.x;
  const int c0 = t % gm.TC, sub = t / gm.TC;
  const int cg = gm.C / gm.groups;
  float s1[kGnMaxJ], s2[kGnMaxJ], mean[kGnMaxJ], rstd[kGnMaxJ];
#pragma unroll
  for (int j = 0; j < kGnMaxJ; ++j) {
    s1[j] = s2[j] = mean[j] = rstd[j] = 0.f;
    if (j < gm.J) {
      const size_t sg = (size_t)n * gm.groups + (c0 + j * gm.TC) / cg;
      mean[j] = stats[2 * sg];
      rstd[j] = stats[2 * sg + 1];
    }
  }
  for (int ch = blockIdx.x; ch < gm.nchunks; ch += gridDim.x) {
    const int p1 = min(ch * kGnChunk + kGnChunk, gm.HW);
    for (int p = ch * kGnChunk + sub; p < p1; p += gm.SUB) {
      const size_t base = ((size_t)n * gm.HW + p) * gm.C;
#pragma unroll
      for (int j = 0; j < kGnMaxJ; ++j) {
        if (j >= gm.J) break;
        const size_t i = base + c0 + j * gm.TC;
        const float dz = gn_dz(dy, y, i);
        s1[j] += dz;
        s2[j] = fmaf(dz, (x[i] - mean[j]) * rstd[j], s2[j]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < kGnMaxJ; ++j) {
    sh[t][j][0] = s1[j];
    sh[t][j][1] = s2[j];
  }
  __syncthreads();
  for (int c = t; c < gm.C; c += kGnThreads) {
    float a = 0.f, b = 0.f;
    for (int u = 0; u < gm.SUB; ++u) {
      a += sh[u * gm.TC + c % gm.TC][c / gm.TC][0];
      b += sh[u * gm.TC + c % gm.TC][c / gm.TC][1];
    }
    float* o = part + (((size_t)n * gridDim.x + blockIdx.x) * gm.C + c) * 2;
    o[0] = a;
    o[1] = b;
  }
}

// per image: chan[n][c] = (sum dz, sum dz xhat) over the CTAs in order (dshift[n][c] = the first), then per group
// coef[n][g] = (sum_c gamma_c chan_c.0, sum_c gamma_c chan_c.1) in channel order
__global__ void gn_bwd_finalize_kernel(const float* __restrict__ part, int nparts, const float* __restrict__ gamma,
                                       int C, int groups, float* __restrict__ chan, float* __restrict__ coef,
                                       float* __restrict__ dshift) {
  const int n = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float a = 0.f, b = 0.f;
    for (int k = 0; k < nparts; ++k) {
      const float* p = part + (((size_t)n * nparts + k) * C + c) * 2;
      a += p[0];
      b += p[1];
    }
    chan[((size_t)n * C + c) * 2] = a;
    chan[((size_t)n * C + c) * 2 + 1] = b;
    if (dshift) dshift[(size_t)n * C + c] = a;
  }
  __syncthreads();
  const int cg = C / groups;
  for (int g = threadIdx.x; g < groups; g += blockDim.x) {
    float A = 0.f, B = 0.f;
    for (int c = g * cg; c < (g + 1) * cg; ++c) {
      A = fmaf(gamma[c], chan[((size_t)n * C + c) * 2], A);
      B = fmaf(gamma[c], chan[((size_t)n * C + c) * 2 + 1], B);
    }
    coef[((size_t)n * groups + g) * 2] = A;
    coef[((size_t)n * groups + g) * 2 + 1] = B;
  }
}

// dgamma[c] = sum_n chan[n][c].1, dbeta[c] = sum_n chan[n][c].0, images in order
__global__ void gn_bwd_param_kernel(const float* __restrict__ chan, int N, int C, float* __restrict__ dgamma,
                                    float* __restrict__ dbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float a = 0.f, b = 0.f;
  for (int n = 0; n < N; ++n) {
    a += chan[((size_t)n * C + c) * 2];
    b += chan[((size_t)n * C + c) * 2 + 1];
  }
  if (dbeta) dbeta[c] = a;
  if (dgamma) dgamma[c] = b;
}

// dx = rstd (gamma dz - (A + xhat B) / M), M = HW C / G
__global__ void __launch_bounds__(kGnThreads)
gn_bwd_dx_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ y,
                 const float* __restrict__ stats, const float* __restrict__ coef, const float* __restrict__ gamma,
                 MapGeom gm, float* __restrict__ dx) {
  const int n = blockIdx.y, t = threadIdx.x;
  const int c0 = t % gm.TC, sub = t / gm.TC;
  const int cg = gm.C / gm.groups;
  const float invM = 1.f / ((float)gm.HW * (float)cg);
  float mean[kGnMaxJ], rstd[kGnMaxJ], A[kGnMaxJ], B[kGnMaxJ], gam[kGnMaxJ];
#pragma unroll
  for (int j = 0; j < kGnMaxJ; ++j) {
    if (j >= gm.J) break;
    const int c = c0 + j * gm.TC;
    const size_t sg = (size_t)n * gm.groups + c / cg;
    mean[j] = stats[2 * sg];
    rstd[j] = stats[2 * sg + 1];
    A[j] = coef[2 * sg];
    B[j] = coef[2 * sg + 1];
    gam[j] = gamma[c];
  }
  for (int ch = blockIdx.x; ch < gm.nchunks; ch += gridDim.x) {
    const int p1 = min(ch * kGnChunk + kGnChunk, gm.HW);
    for (int p = ch * kGnChunk + sub; p < p1; p += gm.SUB) {
      const size_t base = ((size_t)n * gm.HW + p) * gm.C;
#pragma unroll
      for (int j = 0; j < kGnMaxJ; ++j) {
        if (j >= gm.J) break;
        const size_t i = base + c0 + j * gm.TC;
        const float xh = (x[i] - mean[j]) * rstd[j];
        dx[i] = rstd[j] * (gam[j] * gn_dz(dy, y, i) - (A[j] + xh * B[j]) * invM);
      }
    }
  }
}

// dres[n][hr][wr][c] = sum of dz over the 2x2 pixels that read residual pixel (hr, wr)
__global__ void gn_bwd_res_up2_kernel(const float* __restrict__ dy, const float* __restrict__ y, int N, int H, int W,
                                      int C, float* __restrict__ dres) {
  const int Hr = H / 2, Wr = W / 2;
  const size_t total = (size_t)N * Hr * Wr * C;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const size_t q = i / C;
    const int wr = (int)(q % Wr), hr = (int)(q / Wr % Hr);
    const size_t n = q / ((size_t)Wr * Hr);
    float s = 0.f;
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 2; ++b) s += gn_dz(dy, y, ((n * H + 2 * hr + a) * W + 2 * wr + b) * C + c);
    dres[i] = s;
  }
}

int map_blocks(const MapGeom& gm, int limit) { return gm.nchunks < limit ? gm.nchunks : limit; }

bool map_ok(int N, int C, int H, int W, int groups) {
  if (N <= 0 || C <= 0 || H <= 0 || W <= 0 || groups <= 0 || C % groups) return false;
  if (C > kGnMaxC || N > 65535) return false;
  const int TC = C < kGnThreads ? C : kGnThreads;
  return kGnThreads % TC == 0 && C % TC == 0;
}

}  // namespace
}  // namespace ups

extern "C" int upsnet_group_norm_workspace_bytes(int N, int C, int H, int W, int groups, size_t* bytes) {
  using namespace ups;
  if (!bytes) return UPSNET_E_BADARG;
  if (!map_ok(N, C, H, W, groups)) return UPSNET_E_UNSUPPORTED;
  const MapGeom gm = map_geom(C, H, W, groups);
  *bytes = (size_t)N * groups * map_blocks(gm, kGnMaxBlocks) * 3 * sizeof(float);
  return 0;
}

extern "C" int upsnet_group_norm_forward(const void* x, const float* gamma, const float* beta, const float* shift,
                                         const void* residual, void* y, float* stats, int N, int C, int H, int W,
                                         int groups, float eps, int dtype, int flags, void* workspace,
                                         size_t workspace_bytes, void* stream) {
  using namespace ups;
  if (!x || !gamma || !beta || !y || !stats || !workspace) return UPSNET_E_BADARG;
  if (dtype != UPSNET_DTYPE_F32 && dtype != UPSNET_DTYPE_BF16 && dtype != UPSNET_DTYPE_PAIR) return UPSNET_E_BADARG;
  if (!map_ok(N, C, H, W, groups)) return UPSNET_E_UNSUPPORTED;
  if (((flags & UPSNET_EPI_RES_UP2) != 0) != (residual != nullptr)) return UPSNET_E_BADARG;
  if (residual && (H % 2 || W % 2)) return UPSNET_E_UNSUPPORTED;
  size_t need = 0;
  upsnet_group_norm_workspace_bytes(N, C, H, W, groups, &need);
  if (workspace_bytes < need) return UPSNET_E_WORKSPACE;
  const MapGeom gm = map_geom(C, H, W, groups);
  const int nb = map_blocks(gm, kGnMaxBlocks);
  cudaStream_t s = (cudaStream_t)stream;
  float* part = static_cast<float*>(workspace);
  gn_stats_kernel<<<dim3(nb, N), kGnThreads, 0, s>>>(x, dtype, gm, part);
  UPS_CHECK_LAUNCH();
  const int total = N * groups;
  gn_finalize_kernel<<<ceil_div(total, 8), 256, 0, s>>>(part, nb, total, eps, stats);
  UPS_CHECK_LAUNCH();
  const int na = ceil_div(2 * num_sms() * 4, N) < gm.nchunks ? ceil_div(2 * num_sms() * 4, N) : gm.nchunks;
  gn_apply_kernel<<<dim3(na, N), kGnThreads, 0, s>>>(x, stats, gamma, beta, shift, residual, y, dtype, gm, flags);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_group_norm_rows(const void* x, const float* gamma, const float* beta, void* y, int R, int C,
                                      int HW, int groups, float eps, int dtype, int flags, const int* n_dev,
                                      void* stream) {
  using namespace ups;
  if (!x || !gamma || !beta || !y || R < 0 || C <= 0 || HW <= 0 || groups <= 0 || C % groups) return UPSNET_E_BADARG;
  if (dtype != UPSNET_DTYPE_F32 && dtype != UPSNET_DTYPE_BF16 && dtype != UPSNET_DTYPE_PAIR) return UPSNET_E_BADARG;
  if (flags & ~UPSNET_EPI_RELU) return UPSNET_E_BADARG;
  if (R == 0) return 0;
  const long long warps = (long long)R * groups;
  if (warps > (long long)8 * 0x7fffffff) return UPSNET_E_UNSUPPORTED;
  gn_rows_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, (cudaStream_t)stream>>>(x, gamma, beta, y, R, C, HW, groups,
                                                                                eps, dtype, flags, n_dev);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_group_norm_backward_workspace_bytes(int N, int C, int H, int W, int groups, size_t* bytes) {
  using namespace ups;
  if (!bytes) return UPSNET_E_BADARG;
  if (!map_ok(N, C, H, W, groups)) return UPSNET_E_UNSUPPORTED;
  const MapGeom gm = map_geom(C, H, W, groups);
  const size_t nb = (size_t)map_blocks(gm, kGnMaxBlocks);
  *bytes = ((size_t)N * nb * C * 2 + (size_t)N * C * 2 + (size_t)N * groups * 2) * sizeof(float);
  return 0;
}

extern "C" int upsnet_group_norm_backward(const float* dy, const float* x, const float* y, const float* stats,
                                          const float* gamma, float* dx, float* dgamma, float* dbeta, float* dshift,
                                          float* dres, int N, int C, int H, int W, int groups, int flags,
                                          void* workspace, size_t workspace_bytes, void* stream) {
  using namespace ups;
  if (!dy || !x || !stats || !gamma || !dx || !workspace) return UPSNET_E_BADARG;
  if (((flags & UPSNET_EPI_RELU) != 0) != (y != nullptr)) return UPSNET_E_BADARG;
  if (dres && !(flags & UPSNET_EPI_RES_UP2)) return UPSNET_E_BADARG;
  if (!map_ok(N, C, H, W, groups)) return UPSNET_E_UNSUPPORTED;
  if (dres && (H % 2 || W % 2)) return UPSNET_E_UNSUPPORTED;
  size_t need = 0;
  upsnet_group_norm_backward_workspace_bytes(N, C, H, W, groups, &need);
  if (workspace_bytes < need) return UPSNET_E_WORKSPACE;
  const MapGeom gm = map_geom(C, H, W, groups);
  const int nb = map_blocks(gm, kGnMaxBlocks);
  cudaStream_t s = (cudaStream_t)stream;
  float* part = static_cast<float*>(workspace);
  float* chan = part + (size_t)N * nb * C * 2;
  float* coef = chan + (size_t)N * C * 2;
  gn_bwd_reduce_kernel<<<dim3(nb, N), kGnThreads, 0, s>>>(dy, x, y, stats, gm, part);
  UPS_CHECK_LAUNCH();
  gn_bwd_finalize_kernel<<<N, 256, 0, s>>>(part, nb, gamma, C, groups, chan, coef, dshift);
  UPS_CHECK_LAUNCH();
  if (dgamma || dbeta) {
    gn_bwd_param_kernel<<<ceil_div(C, 256), 256, 0, s>>>(chan, N, C, dgamma, dbeta);
    UPS_CHECK_LAUNCH();
  }
  gn_bwd_dx_kernel<<<dim3(nb, N), kGnThreads, 0, s>>>(dy, x, y, stats, coef, gamma, gm, dx);
  UPS_CHECK_LAUNCH();
  if (dres) {
    const size_t total = (size_t)N * (H / 2) * (W / 2) * C;
    const size_t blocks = (total + 255) / 256 < 65535 ? (total + 255) / 256 : 65535;
    gn_bwd_res_up2_kernel<<<(unsigned)blocks, 256, 0, s>>>(dy, y, N, H, W, C, dres);
    UPS_CHECK_LAUNCH();
  }
  return 0;
}
