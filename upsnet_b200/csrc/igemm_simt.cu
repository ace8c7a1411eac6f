// igemm_simt.cu -- fp32 implicit-GEMM convolution / deformable convolution (v1, v2) on CUDA
// cores: the UPSNET_PREC_FP32_SIMT path.  One kernel covers dense k x k convolutions
// (models/resnet.py, fpn.py, rpn.py, rcnn.py), fully-connected layers (1x1 on a 1x1 map) and the
// fused deformable im2col + GEMM (+ bias / residual / ReLU) that replaces
//   deformable_im2col (operators/src/deform_conv_kernel.cu:194-242) -> col buffer in HBM ->
//   torch.mm (operators/functions/deform_conv.py:52-54) -> bias add
// The column operand is produced in shared memory straight from x and never touches HBM
// (the reference writes+reads 1.2 GB for the first semantic-head layer at 1024x2048).
//
// GEMM view: Y[co][p] = sum_k Wt[co][k] * col[k][p],  k = c*kh*kw + tap (reference weight
// layout [Cout, Cin*kh*kw]), p = flattened (image, ho, wo).  CTA tile 64 (co) x 128 (p), BK=16,
// 256 threads, 8x4 register tile, double-buffered smem, per-tile sample table: for every
// (tap, pixel) the four bilinear corner offsets + weights are computed ONCE (they do not
// depend on the channel) and reused for all Cin channels of the deformable group.
// NCHW fp32 in/out like the reference.  This path is bounded by the fp32 FFMA rate, not by
// tensor cores; the wgmma path lives in igemm_tc.cu.
#include "common.cuh"

namespace ups {

constexpr int TM = 64, TN = 128, BK = 16, TMP = TM + 4, NT = 256;

struct ConvParams {
  const float* x; const float* offset; const float* mask; const float* weight;
  const float* bias; const float* residual; float* y;
  int N, Cin, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, dg, Ho, Wo, relu;
};

template <bool DEFORM>
__global__ void __launch_bounds__(NT)
igemm_simt_kernel(const ConvParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int KHW = p.kh * p.kw;
  const int HoWo = p.Ho * p.Wo;
  const long long Ptot = (long long)p.N * HoWo;
  const int K = p.Cin * KHW;
  const int cpg = p.Cin / p.dg;
  const size_t HW = (size_t)p.H * p.W;

  float* As = reinterpret_cast<float*>(smem_raw);                 // [2][BK][TMP]
  float* Bs = As + 2 * BK * TMP;                                  // [2][BK][TN]
  long long* xbase = reinterpret_cast<long long*>(Bs + 2 * BK * TN);  // [TN] image base offset (-1: no pixel)
  unsigned char* tbl_raw = reinterpret_cast<unsigned char*>(xbase + TN);
  float4* tw = reinterpret_cast<float4*>(tbl_raw);                // DEFORM: [KHW][TN] weights
  int4* to = reinterpret_cast<int4*>(tw + (DEFORM ? KHW * TN : 0));   // DEFORM: [KHW][TN] offsets
  int* ti = reinterpret_cast<int*>(tbl_raw);                      // !DEFORM: [KHW][TN] offset or -1

  const int tid = threadIdx.x;
  const long long p0 = (long long)blockIdx.x * TN;
  const int co0 = blockIdx.y * TM;

  for (int pl = tid; pl < TN; pl += NT) {
    const long long pg = p0 + pl;
    xbase[pl] = pg < Ptot ? (long long)(pg / HoWo) * p.Cin * (long long)HW : -1;
  }

  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const int a_co = tid >> 2, a_kq = (tid & 3) * 4;   // A loader: 4 consecutive k of one co
  const int b_pl = tid & (TN - 1), b_kb = (tid >> 7) * 8;  // B loader: 8 consecutive k of one pixel
  const int tx = tid & 31, ty = tid >> 5;
  const bool a_vec = ((K & 3) == 0) && (((cpg * KHW) & 3) == 0) && ((((uintptr_t)p.weight) & 15) == 0);

  for (int g = 0; g < p.dg; ++g) {
    __syncthreads();  // everyone done with the previous group's table / smem tiles
    // ---------------- per-(tile, group) sample table ----------------
    for (int e = tid; e < KHW * TN; e += NT) {
      const int tap = e / TN, pl = e - tap * TN;
      const long long pg = p0 + pl;
      const int ki = tap / p.kw, kj = tap - ki * p.kw;
      if (DEFORM) {
        float4 wv = make_float4(0.f, 0.f, 0.f, 0.f);
        int4 ov = make_int4(0, 0, 0, 0);
        if (pg < Ptot) {
          const int n = (int)(pg / HoWo), pp = (int)(pg - (long long)n * HoWo);
          const int ho = pp / p.Wo, wo = pp - ho * p.Wo;
          const float* offp = p.offset + ((size_t)(n * p.dg + g) * 2 * KHW + 2 * tap) * HoWo + pp;
          const float oh = __ldg(offp), ow = __ldg(offp + HoWo);
          const float h = (float)(ho * p.sh - p.ph + ki * p.dh) + oh;
          const float w = (float)(wo * p.sw - p.pw + kj * p.dw) + ow;
          if (h > -1.f && w > -1.f && h < (float)p.H && w < (float)p.W) {
            const int hl = (int)floorf(h), wl = (int)floorf(w), hh = hl + 1, wh = wl + 1;
            const float lh = h - hl, lw = w - wl, ch = 1.f - lh, cw = 1.f - lw;
            const bool t_ok = hl >= 0, b_ok = hh <= p.H - 1, l_ok = wl >= 0, r_ok = wh <= p.W - 1;
            float m = 1.f;
            if (p.mask) m = __ldg(p.mask + ((size_t)(n * p.dg + g) * KHW + tap) * HoWo + pp);
            wv.x = (t_ok && l_ok) ? ch * cw * m : 0.f;
            wv.y = (t_ok && r_ok) ? ch * lw * m : 0.f;
            wv.z = (b_ok && l_ok) ? lh * cw * m : 0.f;
            wv.w = (b_ok && r_ok) ? lh * lw * m : 0.f;
            ov.x = (t_ok && l_ok) ? hl * p.W + wl : 0;
            ov.y = (t_ok && r_ok) ? hl * p.W + wh : 0;
            ov.z = (b_ok && l_ok) ? hh * p.W + wl : 0;
            ov.w = (b_ok && r_ok) ? hh * p.W + wh : 0;
          }
        }
        tw[e] = wv;
        to[e] = ov;
      } else {
        int o = -1;
        if (pg < Ptot) {
          const int n = (int)(pg / HoWo), pp = (int)(pg - (long long)n * HoWo);
          const int ho = pp / p.Wo, wo = pp - ho * p.Wo;
          const int hi = ho * p.sh - p.ph + ki * p.dh, wi = wo * p.sw - p.pw + kj * p.dw;
          if (hi >= 0 && hi < p.H && wi >= 0 && wi < p.W) o = hi * p.W + wi;
        }
        ti[e] = o;
      }
    }
    __syncthreads();

    const int kbeg = g * cpg * KHW, kend = (g + 1) * cpg * KHW;
    const int ntiles = ceil_div(kend - kbeg, BK);
    float a_reg[4], b_reg[8];

    auto load_tile = [&](int t) {
      const int k0 = kbeg + t * BK;
      // ---- A (weights) ----
      const int co = co0 + a_co;
      const int ka = k0 + a_kq;
      if (a_vec && co < p.Cout && ka + 3 < kend) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(p.weight + (size_t)co * K + ka));
        a_reg[0] = v.x; a_reg[1] = v.y; a_reg[2] = v.z; a_reg[3] = v.w;
      } else {
#pragma unroll
        for (int u = 0; u < 4; ++u)
          a_reg[u] = (co < p.Cout && ka + u < kend) ? __ldg(p.weight + (size_t)co * K + ka + u) : 0.f;
      }
      // ---- B (gathered column operand) ----
      const long long xb = xbase[b_pl];
      int kk = k0 + b_kb;
      int c = kk / KHW, tap = kk - c * KHW;
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        float v = 0.f;
        if (xb >= 0 && kk < kend) {
          const float* xc = p.x + xb + (size_t)c * HW;
          if (DEFORM) {
            const float4 wv = tw[tap * TN + b_pl];
            const int4 ov = to[tap * TN + b_pl];
            v = wv.x * __ldg(xc + ov.x) + wv.y * __ldg(xc + ov.y) + wv.z * __ldg(xc + ov.z) +
                wv.w * __ldg(xc + ov.w);
          } else {
            const int o = ti[tap * TN + b_pl];
            if (o >= 0) v = __ldg(xc + o);
          }
        }
        b_reg[u] = v;
        ++kk;
        if (++tap == KHW) { tap = 0; ++c; }
      }
    };
    auto store_tile = [&](int buf) {
#pragma unroll
      for (int u = 0; u < 4; ++u) As[(buf * BK + a_kq + u) * TMP + a_co] = a_reg[u];
#pragma unroll
      for (int u = 0; u < 8; ++u) Bs[(buf * BK + b_kb + u) * TN + b_pl] = b_reg[u];
    };

    load_tile(0);
    store_tile(0);
    __syncthreads();
    for (int t = 0; t < ntiles; ++t) {
      const int buf = t & 1;
      if (t + 1 < ntiles) load_tile(t + 1);
#pragma unroll
      for (int kk = 0; kk < BK; ++kk) {
        const float4 a0 = *reinterpret_cast<const float4*>(&As[(buf * BK + kk) * TMP + ty * 8]);
        const float4 a1 = *reinterpret_cast<const float4*>(&As[(buf * BK + kk) * TMP + ty * 8 + 4]);
        const float4 b = *reinterpret_cast<const float4*>(&Bs[(buf * BK + kk) * TN + tx * 4]);
        const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
      if (t + 1 < ntiles) store_tile(buf ^ 1);
      __syncthreads();
    }
  }

  // ---------------- epilogue: bias, residual, ReLU ----------------
  const long long pg0 = p0 + tx * 4;
  const bool vec_ok = ((HoWo & 3) == 0) && (pg0 + 3 < Ptot) && ((((uintptr_t)p.y) & 15) == 0) &&
                      (!p.residual || ((((uintptr_t)p.residual) & 15) == 0));
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int co = co0 + ty * 8 + i;
    if (co >= p.Cout) continue;
    const float bv = p.bias ? __ldg(p.bias + co) : 0.f;
    if (vec_ok) {
      const int n = (int)(pg0 / HoWo), pp = (int)(pg0 - (long long)n * HoWo);
      const size_t o = ((size_t)n * p.Cout + co) * HoWo + pp;
      float4 v = make_float4(acc[i][0] + bv, acc[i][1] + bv, acc[i][2] + bv, acc[i][3] + bv);
      if (p.residual) {
        const float4 r = __ldg(reinterpret_cast<const float4*>(p.residual + o));
        v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
      }
      if (p.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
      *reinterpret_cast<float4*>(p.y + o) = v;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const long long pg = pg0 + j;
        if (pg >= Ptot) continue;
        const int n = (int)(pg / HoWo), pp = (int)(pg - (long long)n * HoWo);
        const size_t o = ((size_t)n * p.Cout + co) * HoWo + pp;
        float v = acc[i][j] + bv;
        if (p.residual) v += __ldg(p.residual + o);
        if (p.relu) v = fmaxf(v, 0.f);
        p.y[o] = v;
      }
    }
  }
}

static size_t simt_smem_bytes(bool deform, int KHW) {
  size_t b = sizeof(float) * (2 * BK * TMP + 2 * BK * TN) + sizeof(long long) * TN;
  b += deform ? (size_t)KHW * TN * (sizeof(float4) + sizeof(int4)) : (size_t)KHW * TN * sizeof(int);
  return b;
}

int launch_igemm_simt(const ConvParams& p, cudaStream_t stream) {
  const bool deform = p.offset != nullptr;
  const int KHW = p.kh * p.kw;
  const size_t smem = simt_smem_bytes(deform, KHW);
  if (smem > 227 * 1024) return UPSNET_E_UNSUPPORTED;
  const long long Ptot = (long long)p.N * p.Ho * p.Wo;
  if (Ptot <= 0) return 0;
  const long long gx = (Ptot + TN - 1) / TN;
  if (gx > 2147483647LL) return UPSNET_E_UNSUPPORTED;
  dim3 grid((unsigned)gx, (unsigned)ceil_div(p.Cout, TM));
  static ups::PerDeviceOnce configured;
  if (configured.need()) {
    UPS_CUDA(cudaFuncSetAttribute(igemm_simt_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    UPS_CUDA(cudaFuncSetAttribute(igemm_simt_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  }
  if (deform) igemm_simt_kernel<true><<<grid, NT, smem, stream>>>(p);
  else igemm_simt_kernel<false><<<grid, NT, smem, stream>>>(p);
  UPS_CHECK_LAUNCH();
  return 0;
}

}  // namespace ups
