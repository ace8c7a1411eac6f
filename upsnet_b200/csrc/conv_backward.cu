// conv_backward.cu -- backward of the dense convolutions and FC layers (models/{resnet,fpn,rpn,rcnn}.py: autograd's conv
// backward in the reference) for a layer y = act(conv(x, W) + b [+ residual]):
//
//   prepare  dY (fp32, NCHW or NHWC) -> ReLU mask [y > 0] -> g, NHWC, channels zero-padded to Cp = 64 k, stored as hi/lo
//            pairs (bf16x3) or bf16; d bias as per-CTA partials + one fixed-order pass; d residual (g in fp32, or g summed
//            over 2x2 for the FPN top-down residual_up2) in the same pass.  The 2x2 pixel-unshuffle read mode turns the
//            mask branch's ConvTranspose2d(k = 2, s = 2) into the 1x1 conv to 4 C channels, ordered (a, b, c).
//   dgrad    stride 1: dX = conv(g, W') on the forward kernel (upsnet_igemm_forward) with W'[ci][tap][co] =
//            W[co][ci][flipped tap] (upsnet_igemm_pack_weight_dgrad) and padding d (k - 1) - p.  Stride-2 1x1: the same
//            1x1 conv gives W^T g at the even pixels; upsnet_conv_dgrad_scatter2 writes it, and zeros, into dX.
//   wgrad    dW[co][tap][ci] = sum_p g[p][co] x[p s + tap d - pad][ci]: a GEMM with M = Cout, N = Cin, K = pixels, on
//            the boxes the forward loads (64-channel SWIZZLE_128B boxes of g, and of x shifted by the tap, out-of-range
//            pixels zero-filled by TMA; a strided view for stride 2).  In shared memory both tiles are MN-major (the
//            channels are contiguous, the pixels are rows), so wgmma reads them with the transpose bits (WgmmaT).  K is
//            split over CTAs; each writes an fp32 partial tile to the workspace and one pass adds the splits in a fixed
//            order, straight into torch's [Cout, Cin, kh, kw].  No atomics: the same inputs give the same bytes.
#include <cuda.h>
#include <cuda_bf16.h>

#include "common.cuh"
#include "tc_params.cuh"
#include "tc_ptx.cuh"

namespace ups {

// ----------------------------------------------------------------------------------------------
// prepare
// ----------------------------------------------------------------------------------------------
constexpr int GP_THREADS = 256;
constexpr int GP_TILE = 64;        // g pixels x 64 channels per tile
constexpr int GP_MAX_CTAS = 256;   // CTAs along the pixels (per 64-channel slab): the bias partials per channel

struct GradPrep {
  const float* dy; const float* y;
  void* g; float* dres; double* part;
  int N, C, H, W;                  // logical g: [N, H, W, Cg]; dy is [N, C, H, W] (unshuffle: [N, C, 2H, 2W])
  int Cg, Cp;
  int relu, res, up2, unshuffle, dy_nhwc, pair;
  long long NP;                    // g pixels
  int tiles;                       // pixel tiles (up2: 16 coarse pixels x their 2x2 each)
};

// g pixel of row j of tile t
__device__ __forceinline__ long long gp_pixel(const GradPrep& a, int t, int j) {
  if (!a.up2) return (long long)t * GP_TILE + j;
  const long long q = (long long)t * (GP_TILE / 4) + (j >> 2);
  const int Wq = a.W >> 1, Hq = a.H >> 1;
  if (q >= (long long)a.N * Hq * Wq) return a.NP;
  const int wq = (int)(q % Wq), hq = (int)((q / Wq) % Hq), n = (int)(q / ((long long)Wq * Hq));
  return ((long long)n * a.H + 2 * hq + ((j >> 1) & 1)) * a.W + 2 * wq + (j & 1);
}

// element offset in dy of g element (p, c), c < Cg
__device__ __forceinline__ long long gp_dy_index(const GradPrep& a, long long p, int c) {
  const int w = (int)(p % a.W), h = (int)((p / a.W) % a.H), n = (int)(p / ((long long)a.W * a.H));
  if (!a.unshuffle) {
    if (a.dy_nhwc) return p * a.C + c;
    return ((long long)n * a.C + c) * a.H * a.W + (long long)h * a.W + w;
  }
  const int ab = c / a.C, cc = c - ab * a.C;
  const int hy = 2 * h + (ab >> 1), wy = 2 * w + (ab & 1), Hy = 2 * a.H, Wy = 2 * a.W;
  if (a.dy_nhwc) return (((long long)n * Hy + hy) * Wy + wy) * a.C + cc;
  return (((long long)n * a.C + cc) * Hy + hy) * Wy + wy;
}

__global__ void __launch_bounds__(GP_THREADS) grad_prep_kernel(const GradPrep a) {
  __shared__ float t[GP_TILE][GP_TILE + 1];
  const int tid = threadIdx.x;
  const int c0 = blockIdx.y * 64;
  double bsum = 0.0;                                   // threads 0..63: bias partial of channel c0 + tid (fp64: exact enough
                                                       // that d bias is one fp32 rounding of the sum)
  for (int tile = blockIdx.x; tile < a.tiles; tile += gridDim.x) {
    // dy -> smem, coalesced along whichever of pixels / channels is contiguous in dy
#pragma unroll 4
    for (int i = tid; i < GP_TILE * 64; i += GP_THREADS) {
      const bool cfast = a.dy_nhwc;
      const int cc = cfast ? (i & 63) : (i >> 6), j = cfast ? (i >> 6) : (i & 63);
      const long long p = gp_pixel(a, tile, j);
      const int c = c0 + cc;
      float v = 0.f;
      if (p < a.NP && c < a.Cg) v = __ldg(a.dy + gp_dy_index(a, p, c));
      t[j][cc] = v;
    }
    __syncthreads();
    if (a.relu) {   // y is NHWC [NP][Cg]: channel-fast
      for (int i = tid; i < GP_TILE * 64; i += GP_THREADS) {
        const int cc = i & 63, j = i >> 6;
        const long long p = gp_pixel(a, tile, j);
        const int c = c0 + cc;
        if (p < a.NP && c < a.Cg && !(__ldg(a.y + p * a.Cg + c) > 0.f)) t[j][cc] = 0.f;
      }
      __syncthreads();
    }
    if (tid < 64) {
      for (int j = 0; j < GP_TILE; ++j) bsum += (double)t[j][tid];
    }
    // g: 16-byte vectors of 8 channels (hi plane, lo plane)
    for (int i = tid; i < GP_TILE * 8; i += GP_THREADS) {
      const int q = i & 7, j = i >> 3;
      const long long p = gp_pixel(a, tile, j);
      if (p >= a.NP) continue;
      float o[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = t[j][8 * q + e];
      if (a.pair) {
        uint4 hi, lo;
        split_pair8(o, hi, lo);
        uint4* row = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(a.g) + p * 2 * a.Cp);
        row[(c0 >> 3) + q] = hi;
        row[((a.Cp + c0) >> 3) + q] = lo;
      } else {
        uint4* row = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(a.g) + p * a.Cp);
        row[(c0 >> 3) + q] = pack_bf16x8(o);
      }
    }
    if (a.res) {
      if (!a.up2) {
        for (int i = tid; i < GP_TILE * 64; i += GP_THREADS) {
          const int cc = i & 63, j = i >> 6;
          const long long p = gp_pixel(a, tile, j);
          if (p < a.NP && c0 + cc < a.Cg) a.dres[p * a.Cg + c0 + cc] = t[j][cc];
        }
      } else {
        const long long NQ = (long long)a.N * (a.H >> 1) * (a.W >> 1);
        for (int i = tid; i < (GP_TILE / 4) * 64; i += GP_THREADS) {
          const int cc = i & 63, jq = i >> 6;
          const long long q = (long long)tile * (GP_TILE / 4) + jq;
          if (q < NQ && c0 + cc < a.Cg)
            a.dres[q * a.Cg + c0 + cc] = ((t[4 * jq][cc] + t[4 * jq + 1][cc]) + t[4 * jq + 2][cc]) + t[4 * jq + 3][cc];
        }
      }
    }
    __syncthreads();
  }
  if (tid < 64 && a.part) a.part[(size_t)blockIdx.x * a.Cp + c0 + tid] = bsum;
}

// dbias[c] = sum over the groups k (unshuffle: the four (a, b)) and the CTAs b, in that fixed order
__global__ void grad_bias_kernel(const double* __restrict__ part, int nblk, int Cp, int C, int groups, float* __restrict__ dbias) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double s = 0.0;
  for (int k = 0; k < groups; ++k)
    for (int b = 0; b < nblk; ++b) s += part[(size_t)b * Cp + k * C + c];
  dbias[c] = (float)s;
}

static void grad_prep_geometry(int N, int C, int H, int W, int flags, int* Cg, int* Cp, long long* NP, int* tiles, int* grid_x) {
  const bool unshuffle = (flags & UPSNET_GRAD_UNSHUFFLE2) != 0, up2 = (flags & UPSNET_GRAD_RES_UP2) != 0;
  *Cg = unshuffle ? 4 * C : C;
  *Cp = (*Cg + 63) / 64 * 64;
  *NP = (long long)N * H * W;
  *tiles = up2 ? (int)(((long long)N * (H / 2) * (W / 2) + GP_TILE / 4 - 1) / (GP_TILE / 4)) : (int)((*NP + GP_TILE - 1) / GP_TILE);
  *grid_x = *tiles < GP_MAX_CTAS ? *tiles : GP_MAX_CTAS;
}

// ----------------------------------------------------------------------------------------------
// dgrad helpers: the flipped / transposed weight pack and the stride-2 scatter
// ----------------------------------------------------------------------------------------------
// packed hi / lo planes [cout_pad(Cin)][KHW][Cp]: (ci, tap, co) = W[co][ci][KHW - 1 - tap], zero for co >= Cout, ci >= Cin
__global__ void pack_weight_dgrad_kernel(const float* __restrict__ w, int Cout, int Cin, int KHW, int Cp, int rows,
                                         uint16_t* __restrict__ hi, uint16_t* __restrict__ lo) {
  const size_t K = (size_t)KHW * Cp, total = (size_t)rows * K;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int ci = (int)(i / K), kk = (int)(i - (size_t)ci * K);
    const int tap = kk / Cp, co = kk - tap * Cp;
    const float v = (co < Cout && ci < Cin) ? w[((size_t)co * Cin + ci) * KHW + (KHW - 1 - tap)] : 0.f;
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    hi[i] = *reinterpret_cast<const uint16_t*>(&h);
    lo[i] = *reinterpret_cast<const uint16_t*>(&l);
  }
}

// dx [N, H, W, C] fp32: dxc[n, h / 2, w / 2, c] at even (h, w), 0 elsewhere; float4 per thread
__global__ void dgrad_scatter2_kernel(const float4* __restrict__ dxc, float4* __restrict__ dx, int N, int H, int W, int Ho,
                                      int Wo, int C4) {
  const long long total = (long long)N * H * W * C4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    const long long p = i / C4;
    const int w = (int)(p % W), h = (int)((p / W) % H), n = (int)(p / ((long long)W * H));
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!(h & 1) && !(w & 1)) v = __ldg(dxc + (((long long)n * Ho + (h >> 1)) * Wo + (w >> 1)) * C4 + c);
    dx[i] = v;
  }
}

// ----------------------------------------------------------------------------------------------
// wgrad
// ----------------------------------------------------------------------------------------------
constexpr int WG_THREADS = 9 * 32;     // warps 0-7: two wgmma warpgroups (Cout rows [64 wg, 64 wg + 64)); warp 8: TMA
constexpr int WG_WARP_TMA = 8;
constexpr int WG_SLAB = 64 * 128;      // 64 pixels x 64 channels of bf16
constexpr int WG_MAX_STAGES = 8;

struct WgradGeom {
  int KHW, kw, ph, pw, dh, dw;
  int bw, bh, bn, tw, th, nb;          // pixel box (bw x bh x bn <= 64 pixels), boxes along W / H, boxes in all
  int mt, nt, splits;                  // Cout / 128 and Cin / 128 tiles (rounded up), K splits
  int Mpad, Npad;
  float* ws;                           // [splits][KHW][Mpad][Npad] fp32 partial tiles
  int stages;
};

// Stage s: A (g) planes [plane][co slab][64 px rows][128 B], then B (x) planes [plane][ci slab][64 px rows][128 B].
template <bool X3>
__global__ void __launch_bounds__(WG_THREADS, 1)
wgrad_kernel(const __grid_constant__ CUtensorMap tm_g, const __grid_constant__ CUtensorMap tm_x, const WgradGeom G) {
  constexpr int P = X3 ? 2 : 1;
  constexpr uint32_t A_BYTES = P * 2 * WG_SLAB, STAGE = 2 * A_BYTES;
  extern __shared__ __align__(1024) uint8_t smem_dyn[];
  const uint32_t raw = smem_u32(smem_dyn);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* sm = smem_dyn + (base - raw);
  const uint32_t bar_full = base, bar_empty = base + 8 * WG_MAX_STAGES;
  const uint32_t st_base = base + 1024;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  const int split = blockIdx.x % G.splits;
  int tile = blockIdx.x / G.splits;
  const int tap = tile % G.KHW; tile /= G.KHW;
  const int nti = tile % G.nt, mti = tile / G.nt;
  const int kb0 = (int)((long long)split * G.nb / G.splits), kb1 = (int)((long long)(split + 1) * G.nb / G.splits);
  const int co0 = mti * 128, ci0 = nti * 128;
  const int ki = tap / G.kw, kj = tap - ki * G.kw;

  // Rows of a slab beyond the box (boxes of fewer than 64 pixels) are never written by TMA: zero the ring once so that
  // they add nothing.
  {
    uint4* z = reinterpret_cast<uint4*>(sm + 1024);
    const int n16 = (int)(STAGE * (uint32_t)G.stages / 16u);
    for (int i = tid; i < n16; i += WG_THREADS) z[i] = make_uint4(0u, 0u, 0u, 0u);
  }
  fence_proxy_async();
  if (tid == 0) {
    for (int s = 0; s < G.stages; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, 8);
    }
    fence_mbar_init();
  } else if (warp == WG_WARP_TMA && lane == 0) {
    prefetch_tmap(&tm_g);
    prefetch_tmap(&tm_x);
  }
  __syncthreads();

  if (warp == WG_WARP_TMA) {
    if (lane == 0) {
      const uint32_t box_bytes = (uint32_t)(G.bw * G.bh * G.bn) * 128u;
      uint32_t s = 0, ph = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        const int bx = kb % G.tw, by = (kb / G.tw) % G.th, bz = kb / (G.tw * G.th);
        const int w0 = bx * G.bw, h0 = by * G.bh, n0 = bz * G.bn;
        const uint32_t bf = bar_full + 8 * s, dst = st_base + s * STAGE;
        mbar_wait(bar_empty + 8 * s, ph ^ 1u);
        mbar_arrive_expect_tx(bf, 4u * P * box_bytes);
#pragma unroll
        for (int pl = 0; pl < P; ++pl)
#pragma unroll
          for (int sl = 0; sl < 2; ++sl) {
            tma_load_5d(dst + (uint32_t)(pl * 2 + sl) * WG_SLAB, &tm_g, bf, co0 + 64 * sl, pl, w0, h0, n0);
            tma_load_5d(dst + A_BYTES + (uint32_t)(pl * 2 + sl) * WG_SLAB, &tm_x, bf, ci0 + 64 * sl, pl,
                        w0 + kj * G.dw - G.pw, h0 + ki * G.dh - G.ph, n0);
          }
        if (++s == (uint32_t)G.stages) { s = 0; ph ^= 1u; }
      }
    }
    __syncwarp();
    return;
  }

  // consumers
  const int wg = warp >> 2;
  const uint32_t dhi = wg_desc_hi(1024);
  float d[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) d[i] = 0.f;
  uint32_t s = 0, ph = 0;
  int prev = -1;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(bar_full + 8 * s, ph);
    const uint32_t st = st_base + s * STAGE;
    // A: this warpgroup's 64-channel g slab; B: both x slabs, 64-channel blocks WG_SLAB apart (leading byte offset)
    const uint32_t a_hi = wg_desc_mn_lo(st + (uint32_t)wg * WG_SLAB, WG_SLAB);
    const uint32_t b_hi = wg_desc_mn_lo(st + A_BYTES, WG_SLAB);
    wgmma_fence();
#pragma unroll
    for (uint32_t k = 0; k < 4; ++k) {             // 16 pixel rows = 2 KB = 128 descriptor units
      if constexpr (X3) {                          // lo*hi + hi*lo + hi*hi, as the forward
        const uint32_t a_lo = a_hi + (2u * WG_SLAB >> 4), b_lo = b_hi + (2u * WG_SLAB >> 4);
        WgmmaT<128>::mma(d, wg_desc(a_lo + 128 * k, dhi), wg_desc(b_hi + 128 * k, dhi), 1u);
        WgmmaT<128>::mma(d, wg_desc(a_hi + 128 * k, dhi), wg_desc(b_lo + 128 * k, dhi), 1u);
        WgmmaT<128>::mma(d, wg_desc(a_hi + 128 * k, dhi), wg_desc(b_hi + 128 * k, dhi), 1u);
      } else {
        WgmmaT<128>::mma(d, wg_desc(a_hi + 128 * k, dhi), wg_desc(b_hi + 128 * k, dhi), 1u);
      }
    }
    wgmma_commit();
    wgmma_wait<1>();
    wgmma_fence_acc(d);
    if (prev >= 0 && lane == 0) mbar_arrive(bar_empty + 8 * prev);
    prev = (int)s;
    if (++s == (uint32_t)G.stages) { s = 0; ph ^= 1u; }
  }
  wgmma_wait<0>();
  wgmma_fence_acc(d);
  // fragment -> partial tile: d[4 i + 2 h + e] is Cout row 16 (warp & 3) + lane / 4 + 8 h, Cin column 8 i + 2 (lane & 3) + e
  float* out = G.ws + ((size_t)(split * G.KHW + tap) * G.Mpad + co0 + wg * 64) * G.Npad + ci0;
#pragma unroll
  for (int i = 0; i < 16; ++i)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = 16 * (warp & 3) + (lane >> 2) + 8 * h, c = 8 * i + 2 * (lane & 3);
      *reinterpret_cast<float2*>(out + (size_t)r * G.Npad + c) = make_float2(d[4 * i + 2 * h], d[4 * i + 2 * h + 1]);
    }
}

// dW from the partial tiles, splits added in order.  deconv2: the 1x1 conv to 4 C channels (a, b, c) of a
// ConvTranspose2d(k = 2, s = 2), written as its weight [Cin][C][2][2].
__global__ void wgrad_reduce_kernel(const float* __restrict__ ws, int splits, int KHW, int Mpad, int Npad, int Cout, int Cin,
                                    int deconv2, float* __restrict__ dw) {
  const long long total = (long long)Cout * Cin * KHW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int co, ci, tap;
    if (deconv2) {   // i = ((ci * C + c) * 2 + a) * 2 + b, co = (2 a + b) C + c
      const int C = Cout / 4, ab = (int)(i & 3);
      const long long r = i >> 2;
      const int c = (int)(r % C);
      ci = (int)(r / C); co = ab * C + c; tap = 0;
    } else {
      tap = (int)(i % KHW);
      const long long r = i / KHW;
      ci = (int)(r % Cin); co = (int)(r / Cin);
    }
    float s = 0.f;
    for (int k = 0; k < splits; ++k) s += ws[(((size_t)k * KHW + tap) * Mpad + co) * Npad + ci];
    dw[i] = s;
  }
}

// 5-D bf16 map (channels, plane, w, h, n) with explicit byte strides of dims 1..4; box (64, 1, bw, bh, bn)
static bool encode_grad_map(CUtensorMap* tm, const void* ptr, int C, int planes, int W, int H, int N, cuuint64_t s1,
                            cuuint64_t s2, cuuint64_t s3, cuuint64_t s4, int bw, int bh, int bn) {
  EncodeTiledFn enc = tma_encoder();
  if (!enc) return false;
  const cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)planes, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t strides[4] = {s1, s2, s3, s4};
  const cuuint32_t box[5] = {64, 1, (cuuint32_t)bw, (cuuint32_t)bh, (cuuint32_t)bn};
  const cuuint32_t es[5] = {1, 1, 1, 1, 1};
  return enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(ptr), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Pixel box of at most 64 output pixels: fewest boxes, then the fullest box, then the widest rows.
static void wgrad_pick_box(int N, int Ho, int Wo, int* bw_o, int* bh_o, int* bn_o) {
  long long best = -1;
  int bbw = 1, bbh = 1, bbn = 1, bfill = 0;
  for (int bw = 1; bw <= (Wo < 64 ? Wo : 64); ++bw) {
    if (Wo > 16 && (bw & (bw - 1))) continue;
    for (int bh = 1; bh <= (64 / bw < Ho ? 64 / bw : Ho); ++bh) {
      int bn = 64 / (bw * bh);
      if (bn > N) bn = N;
      const long long boxes = (long long)((Wo + bw - 1) / bw) * ((Ho + bh - 1) / bh) * ((N + bn - 1) / bn);
      const int fill = bw * bh * bn;
      if (best < 0 || boxes < best || (boxes == best && (fill > bfill || (fill == bfill && bw > bbw)))) {
        best = boxes; bbw = bw; bbh = bh; bbn = bn; bfill = fill;
      }
    }
  }
  *bw_o = bbw; *bh_o = bbh; *bn_o = bbn;
}

struct WgradPlan {
  WgradGeom g;
  size_t ws_bytes;
};

static int wgrad_plan(int N, int H, int W, int Cin, int Cout, int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw,
                      int precision, WgradPlan* pl) {
  if (N <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0 || kh <= 0 || kw <= 0 || sh <= 0 || sw <= 0 || ph < 0 || pw < 0 ||
      dh <= 0 || dw <= 0)
    return UPSNET_E_BADARG;
  if (precision != UPSNET_PREC_BF16X3 && precision != UPSNET_PREC_BF16) return UPSNET_E_BADARG;
  if ((sh != 1 || sw != 1) && (kh != 1 || kw != 1 || ph != 0 || pw != 0)) return UPSNET_E_UNSUPPORTED;
  if (Cin % 64 || kh * kw > 49) return UPSNET_E_UNSUPPORTED;
  const int Ho = conv_out_size(H, ph, dh, kh, sh), Wo = conv_out_size(W, pw, dw, kw, sw);
  if (Ho <= 0 || Wo <= 0) return UPSNET_E_BADARG;
  WgradGeom& g = pl->g;
  g = WgradGeom{};
  g.KHW = kh * kw; g.kw = kw; g.ph = ph; g.pw = pw; g.dh = dh; g.dw = dw;
  wgrad_pick_box(N, Ho, Wo, &g.bw, &g.bh, &g.bn);
  g.tw = (Wo + g.bw - 1) / g.bw; g.th = (Ho + g.bh - 1) / g.bh;
  const long long nb = (long long)g.tw * g.th * ((N + g.bn - 1) / g.bn);
  if (nb >= (1ll << 31)) return UPSNET_E_UNSUPPORTED;
  g.nb = (int)nb;
  g.mt = (Cout + 127) / 128; g.nt = (Cin + 127) / 128;
  g.Mpad = 128 * g.mt; g.Npad = 128 * g.nt;
  // K splits: about two CTAs per SM over all tiles, at least two boxes per split
  const long long tiles = (long long)g.mt * g.nt * g.KHW;
  long long S = (2LL * num_sms() + tiles - 1) / tiles;
  if (S > g.nb / 2) S = g.nb / 2;
  if (S < 1) S = 1;
  g.splits = (int)S;
  if (tiles * S >= (1ll << 31)) return UPSNET_E_UNSUPPORTED;
  const uint32_t stage = (precision == UPSNET_PREC_BF16X3 ? 2u : 1u) * 4u * WG_SLAB;
  g.stages = (int)((227u * 1024u - 2048u) / stage);
  if (g.stages > WG_MAX_STAGES) g.stages = WG_MAX_STAGES;
  pl->ws_bytes = (size_t)S * g.KHW * g.Mpad * g.Npad * sizeof(float);
  return 0;
}

}  // namespace ups

// ----------------------------------------------------------------------------------------------
// C ABI
// ----------------------------------------------------------------------------------------------
extern "C" int upsnet_conv_grad_prepare_workspace_bytes(int N, int C, int H, int W, int flags, size_t* bytes) {
  if (!bytes || N <= 0 || C <= 0 || H <= 0 || W <= 0) return UPSNET_E_BADARG;
  int Cg, Cp, tiles, gx;
  long long NP;
  ups::grad_prep_geometry(N, C, H, W, flags, &Cg, &Cp, &NP, &tiles, &gx);
  *bytes = (size_t)gx * Cp * sizeof(double);
  return 0;
}

extern "C" int upsnet_conv_grad_prepare(const float* dy, const float* y, void* g, float* dbias, float* dres, int N, int C, int H,
                                        int W, int flags, int precision, void* workspace, size_t workspace_bytes, void* stream) {
  using namespace ups;
  if (!dy || !g || N <= 0 || C <= 0 || H <= 0 || W <= 0) return UPSNET_E_BADARG;
  if (precision != UPSNET_PREC_BF16X3 && precision != UPSNET_PREC_BF16) return UPSNET_E_BADARG;
  GradPrep a{};
  a.relu = (flags & UPSNET_GRAD_RELU) != 0;
  a.up2 = (flags & UPSNET_GRAD_RES_UP2) != 0;
  a.res = dres != nullptr;
  a.unshuffle = (flags & UPSNET_GRAD_UNSHUFFLE2) != 0;
  a.dy_nhwc = (flags & UPSNET_GRAD_DY_NHWC) != 0;
  a.pair = precision == UPSNET_PREC_BF16X3;
  if (a.relu && !y) return UPSNET_E_BADARG;
  if (a.up2 && (!a.res || (H & 1) || (W & 1))) return UPSNET_E_BADARG;
  if (a.unshuffle && a.res) return UPSNET_E_UNSUPPORTED;
  if ((((uintptr_t)g) & 15)) return UPSNET_E_BADARG;
  int gx;
  grad_prep_geometry(N, C, H, W, flags, &a.Cg, &a.Cp, &a.NP, &a.tiles, &gx);
  if (dbias) {
    if (!workspace || workspace_bytes < (size_t)gx * a.Cp * sizeof(double) || (((uintptr_t)workspace) & 7)) return UPSNET_E_WORKSPACE;
  }
  a.dy = dy; a.y = y; a.g = g; a.dres = dres; a.part = dbias ? reinterpret_cast<double*>(workspace) : nullptr;
  a.N = N; a.C = C; a.H = H; a.W = W;
  cudaStream_t st = (cudaStream_t)stream;
  if (a.tiles <= 0) return 0;
  grad_prep_kernel<<<dim3((unsigned)gx, (unsigned)(a.Cp / 64)), GP_THREADS, 0, st>>>(a);
  UPS_CHECK_LAUNCH();
  if (dbias) {
    grad_bias_kernel<<<(C + 127) / 128, 128, 0, st>>>(reinterpret_cast<const double*>(workspace), gx, a.Cp, C,
                                                      a.unshuffle ? 4 : 1, dbias);
    UPS_CHECK_LAUNCH();
  }
  return 0;
}

extern "C" int upsnet_igemm_packed_weight_dgrad_bytes(int Cout, int Cin, int kh, int kw, size_t* bytes) {
  if (!bytes || Cout <= 0 || Cin <= 0 || kh <= 0 || kw <= 0) return UPSNET_E_BADARG;
  if (kh * kw > 49) return UPSNET_E_UNSUPPORTED;
  const int Cp = (Cout + 63) / 64 * 64;
  *bytes = (size_t)2 * ups::cout_pad(Cin) * (size_t)kh * kw * Cp * sizeof(uint16_t);
  return 0;
}

extern "C" int upsnet_igemm_pack_weight_dgrad(const float* weight, int Cout, int Cin, int kh, int kw, void* packed, void* stream) {
  if (!weight || !packed || Cout <= 0 || Cin <= 0 || kh <= 0 || kw <= 0) return UPSNET_E_BADARG;
  if (kh * kw > 49) return UPSNET_E_UNSUPPORTED;
  const int Cp = (Cout + 63) / 64 * 64, rows = ups::cout_pad(Cin), KHW = kh * kw;
  uint16_t* hi = reinterpret_cast<uint16_t*>(packed);
  uint16_t* lo = hi + (size_t)rows * KHW * Cp;
  const size_t total = (size_t)rows * KHW * Cp;
  int blocks = (int)((total + 255) / 256);
  if (blocks > ups::kNumSMs * 16) blocks = ups::kNumSMs * 16;
  ups::pack_weight_dgrad_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(weight, Cout, Cin, KHW, Cp, rows, hi, lo);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_conv_dgrad_scatter2(const float* dxc, float* dx, int N, int H, int W, int C, void* stream) {
  if (!dxc || !dx || N <= 0 || H <= 0 || W <= 0 || C <= 0) return UPSNET_E_BADARG;
  if ((C & 3) || (((uintptr_t)dxc) & 15) || (((uintptr_t)dx) & 15)) return UPSNET_E_UNSUPPORTED;
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const long long total = (long long)N * H * W * (C / 4);
  long long blocks = (total + 255) / 256;
  if (blocks > ups::kNumSMs * 32) blocks = ups::kNumSMs * 32;
  if (total <= 0) return 0;
  ups::dgrad_scatter2_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float4*>(dxc), reinterpret_cast<float4*>(dx), N, H, W, Ho, Wo, C / 4);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_conv_wgrad_workspace_bytes(int N, int H, int W, int Cin, int Cout, int kh, int kw, int stride_h,
                                                 int stride_w, int pad_h, int pad_w, int dil_h, int dil_w, int precision,
                                                 size_t* bytes) {
  if (!bytes) return UPSNET_E_BADARG;
  ups::WgradPlan pl;
  const int rc = ups::wgrad_plan(N, H, W, Cin, Cout, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w, precision, &pl);
  if (rc) return rc;
  *bytes = pl.ws_bytes;
  return 0;
}

extern "C" int upsnet_conv_wgrad(const void* x_nhwc, const void* g, float* dw, int N, int H, int W, int Cin, int Cout, int kh,
                                 int kw, int stride_h, int stride_w, int pad_h, int pad_w, int dil_h, int dil_w, int flags,
                                 int precision, void* workspace, size_t workspace_bytes, void* stream) {
  using namespace ups;
  if (!x_nhwc || !g || !dw) return UPSNET_E_BADARG;
  WgradPlan pl;
  const int rc = wgrad_plan(N, H, W, Cin, Cout, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w, precision, &pl);
  if (rc) return rc;
  const bool deconv2 = (flags & UPSNET_GRAD_UNSHUFFLE2) != 0;
  if (deconv2 && (kh != 1 || kw != 1 || (Cout & 3))) return UPSNET_E_BADARG;
  if (!workspace || workspace_bytes < pl.ws_bytes || (((uintptr_t)workspace) & 15)) return UPSNET_E_WORKSPACE;
  if ((((uintptr_t)x_nhwc) & 15) || (((uintptr_t)g) & 15)) return UPSNET_E_BADARG;
  WgradGeom G = pl.g;
  G.ws = reinterpret_cast<float*>(workspace);
  const bool x3 = precision == UPSNET_PREC_BF16X3;
  const int P = x3 ? 2 : 1;
  const int Ho = conv_out_size(H, pad_h, dil_h, kh, stride_h), Wo = conv_out_size(W, pad_w, dil_w, kw, stride_w);
  const int Cp = (Cout + 63) / 64 * 64;
  CUtensorMap tm_g, tm_x;
  {
    const cuuint64_t e = 2;
    if (!encode_grad_map(&tm_g, g, Cp, P, Wo, Ho, N, Cp * e, (cuuint64_t)P * Cp * e, (cuuint64_t)Wo * P * Cp * e,
                         (cuuint64_t)Ho * Wo * P * Cp * e, G.bw, G.bh, G.bn))
      return UPSNET_E_UNSUPPORTED;
    const bool strided = stride_h != 1 || stride_w != 1;
    const cuuint64_t px = (cuuint64_t)P * Cin * e;
    if (!encode_grad_map(&tm_x, x_nhwc, Cin, P, strided ? Wo : W, strided ? Ho : H, N, Cin * e, px * stride_w,
                         px * W * stride_h, px * W * H, G.bw, G.bh, G.bn))
      return UPSNET_E_UNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const long long ctas = (long long)G.mt * G.nt * G.KHW * G.splits;
  const size_t smem = 1024 + 1024 + (size_t)G.stages * (size_t)P * 4 * WG_SLAB;
  static PerDeviceOnce configured;
  if (configured.need()) {
    UPS_CUDA(cudaFuncSetAttribute(wgrad_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    UPS_CUDA(cudaFuncSetAttribute(wgrad_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  }
  if (x3) wgrad_kernel<true><<<(unsigned)ctas, WG_THREADS, smem, st>>>(tm_g, tm_x, G);
  else wgrad_kernel<false><<<(unsigned)ctas, WG_THREADS, smem, st>>>(tm_g, tm_x, G);
  UPS_CHECK_LAUNCH();
  const long long total = (long long)Cout * Cin * kh * kw;
  long long blocks = (total + 255) / 256;
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  wgrad_reduce_kernel<<<(unsigned)blocks, 256, 0, st>>>(G.ws, G.splits, G.KHW, G.Mpad, G.Npad, Cout, Cin, deconv2 ? 1 : 0, dw);
  UPS_CHECK_LAUNCH();
  return 0;
}
