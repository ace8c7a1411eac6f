// igemm_tc.cu -- wgmma implicit-GEMM convolution / deformable convolution for sm_90a.
//
// One warp-specialised kernel covers the dense k x k convolutions of the backbone / FPN / RPN /
// heads, the fully connected layers and the FUSED deformable conv v1/v2 (im2col never leaves the
// SM; reference: deformable_im2col -> 1.2 GB col buffer -> torch.mm, operators/functions/
// deform_conv.py:44-57 + operators/src/deform_conv_kernel.cu:194-242).
//
//   D[128 pixels x BN couts] (fp32, registers)  +=  A[128 x 64] (bf16, smem)  *  B[BN x 64]^T (bf16, smem)
//
// * A (activations, NHWC fp32 in HBM) is GATHERED by 8 producer warps: for k-block (tap, 64
//   channels) every (pixel,8-channel) item is one or -- when deformable -- four 32-byte reads
//   (the four bilinear corners; weights/offsets come from a per-tile sample table computed once
//   per (tap,pixel), reused by all channels), blended in fp32, converted to bf16 and stored with
//   one 16-byte st.shared into the K-major SWIZZLE_128B layout wgmma consumes.
// * B (weights) is pre-packed once to bf16 [Cout_pad][tap][Cin] and copied by the same warps.
// * One consumer warpgroup issues two wgmma (M=64 each: rows 0-63 and 64-127 of the tile, N=BN,
//   K=16) per 16-column slice with the accumulators in registers; a stage goes back to the producers through an
//   mbarrier once the wgmmas that read it have completed.  At the end of a tile the accumulators
//   are staged through shared memory 32 columns at a time and written out by the same 4 warps
//   (thread = output pixel) while the producers already fill the ring for the next tile
//   (persistent CTAs, static tile schedule).
// * Precision modes: BF16 (one pass) and BF16X3 (x = hi + lo split of both operands, three
//   MMAs: hi*hi + lo*hi + hi*lo; error ~2^-16 relative, i.e. fp32-grade results for the
//   "fp32 logits within 1e-3" contract at 3x the tensor work).
// Roofline: tensor pipe (flops = 2*P*Cout*Cin*kh*kw); the deformable variant is bounded by the
// LSU gather rate of the producers (4 corner reads per element) -- see DESIGN.md.
#include <cuda_bf16.h>
#include <cstdio>

#include "common.cuh"
#include "tc_ptx.cuh"
#include "tc_params.cuh"

namespace ups {

constexpr int TC_BM = 128;         // pixels per tile (UMMA M)
constexpr int TC_BK = 64;          // bf16 elements per k-block row (= 128 bytes, one swizzle span)
constexpr int TC_GROUP = 256;       // producer threads that fill one smem stage together (8 warps)
constexpr int TC_GROUPS = 2;        // producer groups work on alternate k-blocks (two stages in flight)
constexpr int TC_PRODUCERS = TC_GROUP * TC_GROUPS;  // 16 warps
constexpr int TC_CONSUMERS = 128;     // 4 warps = one wgmma warpgroup; in the epilogue thread = tile row
constexpr int TC_EPI_PITCH = 36;      // floats per staged row: 32 columns + 4 pad (16-byte aligned, conflict-free)
constexpr int TC_THREADS = TC_CONSUMERS + TC_PRODUCERS;  // 20 warps
constexpr int TC_MAX_STAGES = 6;
// named barriers (id 0 is __syncthreads): 1 = the producer warps, 2 = the consumer warps



// shared-memory carve-up (offsets from the 1024-aligned base)
struct TcSmem {
  uint32_t bars;      // full[6], empty[6]
  uint32_t rowbase;   // long long [128]
  uint32_t epi;       // accumulator staging: 128 rows x 36 floats (32 columns at a time)
  uint32_t table;     // deform: float4 [KHW][128] + int4 [KHW][128]; dense: int [KHW][128]
  uint32_t stages;    // 1024-aligned
  uint32_t a_bytes, b_bytes, stage_bytes, total;
};
__host__ __device__ inline TcSmem tc_smem_layout(bool deform, int KHW, int BN, int stages, bool x3) {
  TcSmem s;
  s.bars = 0;
  s.rowbase = 256;
  s.epi = s.rowbase + 2 * TC_BM * 8;     // two row-info buffers, then the epilogue staging area
  s.table = s.epi + TC_BM * TC_EPI_PITCH * 4;
  const uint32_t tbytes = deform ? KHW * TC_BM * 32 : KHW * TC_BM * 4;
  s.stages = (uint32_t)((s.table + tbytes + 1023) / 1024 * 1024);
  s.a_bytes = TC_BM * 128;
  s.b_bytes = BN * 128;
  s.stage_bytes = (s.a_bytes + s.b_bytes) * (x3 ? 2 : 1);
  s.total = s.stages + s.stage_bytes * stages;
  return s;
}

// Persistent, warp-specialised kernel.  Roles (20 warps):
//   warps 0-3   consumers: one warpgroup issues wgmma (accumulators in registers), then stages the accumulators
//               through shared memory and applies bias/residual/ReLU and stores (thread = tile row)
//   warps 4-19  producers, two groups of 8 warps filling alternate k-blocks (two smem stages in flight):
//               sample table, B via cp.async, A gather (loads issued first, then bf16 conversion)
// Pipeline: smem ring full[s]/empty[s] (producers <-> consumers) runs across tiles, so the producers fill the
// next tile's stages while the consumers write the previous tile out.
// Tiles: id = blockIdx.x + it*gridDim.x, n-tile fastest (concurrent CTAs share the A rows in L2).
// MODE: 0 = dense (Cin % 64 == 0, NHWC), 1 = deformable, 2 = tiny Cin (stem: NCHW fp32 image, K = kh*kw*Cin
// flattened and zero-padded to a multiple of 64, element-wise gather through a per-k table)
// XM: activation storage of x -- 0 fp32, 1 bf16, 2 hi/lo bf16 pairs (NHWC with 2*Cin channels; always the 3-MMA split)
// BN: N tile (== p.BN), the width of the wgmma instruction and of the register accumulators
template <int MODE, int XM, int BN>
__global__ void __launch_bounds__(TC_THREADS, 1)
igemm_tc_kernel(const TcParams p) {
  constexpr bool XBF16 = XM == 1;
  constexpr bool XPAIR = XM == 2;
  constexpr bool DEFORM = MODE == 1;
  constexpr bool SMALLC = MODE == 2;
  extern __shared__ __align__(1024) uint8_t smem_dyn[];
  const uint32_t raw = smem_u32(smem_dyn);
  const uint32_t base = (raw + 1023u) & ~1023u;   // SWIZZLE_128B stage buffers need 1024-byte alignment
  uint8_t* sm = smem_dyn + (base - raw);

  const int KHW = p.kh * p.kw;
  const bool x3 = p.x3 != 0;
  const TcSmem L = tc_smem_layout(DEFORM, SMALLC ? 2 : KHW, p.BN, p.stages, x3);
  const uint32_t bar_full = base + L.bars, bar_empty = bar_full + 8 * TC_MAX_STAGES;
  long long* rowbase = reinterpret_cast<long long*>(sm + L.rowbase);
  float4* tw = reinterpret_cast<float4*>(sm + L.table);
  int4* to = reinterpret_cast<int4*>(sm + L.table + (DEFORM ? KHW * TC_BM * 16 : 0));
  int* ti = reinterpret_cast<int*>(sm + L.table);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int HoWo = p.Ho * p.Wo;
  const long long Ptot = (long long)p.N * HoWo;
  const int cchunks = SMALLC ? 1 : p.Cin / TC_BK;
  const int Kreal = KHW * p.Cin;
  const int Kp = (Kreal + TC_BK - 1) / TC_BK * TC_BK;      // == Kreal unless SMALLC
  const int num_kb = Kp / TC_BK;
  const int n_tiles = p.Cout_pad / p.BN;
  // M-tile = 128 output pixels.  Dense / stem modes: 128 consecutive pixels of the flattened (n, ho, wo) index.
  // Deformable mode: a 16 x 8 pixel BLOCK of one image -- its nine taps x four corners then revisit ~(16+3) x (8+3)
  // input pixels per channel chunk (27 KB: L1-resident) instead of four 131-pixel row segments.
  // (small maps use 8x8 or 8x4 blocks -- rows past the block stay empty and cost no gather work -- so that more CTAs
  // share the serial k-block chain; the launcher picks the block)
  const int TW = DEFORM ? p.tile_w : 16, TH = DEFORM ? p.tile_h : 8;
  const int tw_shift = TW == 16 ? 4 : 3;
  const int tiles_w = (p.Wo + TW - 1) / TW, tiles_h = (p.Ho + TH - 1) / TH;
  const long long m_tiles = DEFORM ? (long long)p.N * tiles_w * tiles_h : (Ptot + TC_BM - 1) / TC_BM;
  const long long num_tiles = m_tiles * n_tiles;
  // flattened output pixel of row r of M-tile mt, or -1 when the row lies outside the tensor
  auto tile_pixel = [&](long long mt, int r) -> long long {
    if (DEFORM) {
      const int tx = (int)(mt % tiles_w), ty = (int)((mt / tiles_w) % tiles_h), n = (int)(mt / ((long long)tiles_w * tiles_h));
      const int ry = r >> tw_shift;
      const int wo = tx * TW + (r & (TW - 1)), ho = ty * TH + ry;
      return (ry < TH && wo < p.Wo && ho < p.Ho) ? ((long long)n * p.Ho + ho) * p.Wo + wo : -1ll;
    }
    const long long pg = mt * TC_BM + r;
    return pg < Ptot ? pg : -1ll;
  };

  // ---------------- one-time setup ----------------
  if (tid == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(bar_full + 8 * s, TC_GROUP / 32);
      mbar_init(bar_empty + 8 * s, TC_CONSUMERS / 32);   // one arrive per consumer warp
    }
    fence_mbar_init();
  }
  if (SMALLC) {   // per-k table: k -> (dy, dx, channel) packed, -1 for the zero padding of K
    for (int k = tid; k < Kp; k += TC_THREADS) {
      int v = -1;
      if (k < Kreal) {
        const int tap = k / p.Cin, c = k - tap * p.Cin;
        const int ki = tap / p.kw, kj = tap - ki * p.kw;
        v = ((ki * p.dh) << 16) | ((kj * p.dw) << 8) | c;
      }
      ti[k] = v;
    }
  }
  __syncthreads();

  if (warp >= TC_CONSUMERS / 32) {
    // =============================== PRODUCERS ===============================
    const int pt = tid - TC_CONSUMERS;    // 0..511
    const int group = pt / TC_GROUP;      // which alternate k-blocks this thread fills
    const int gt = pt - group * TC_GROUP; // 0..255 inside the group
    const int j = gt & 7;                 // 16-byte chunk (8 channels) inside the 128-byte row
    const int r_first = gt >> 3;          // 32 rows per pass
    uint32_t g0 = 0;                      // ring position of this tile's first k-block
    uint32_t tile_it = 0;
    // bf16 dense mode: both operands travel by cp.async, so the producer keeps ONE k-block outstanding and
    // signals the previous one only after issuing the next (two k-blocks of loads in flight per group).
    const bool deferred = (MODE == 0) && (XBF16 || XPAIR) && p.stages >= 3;
    int pend_s = -1;
    for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const long long mt = tile / n_tiles;
      const int n0 = (int)(tile % n_tiles) * p.BN;
      // Per-tile row info (image, top-left input coordinate of the receptive field) is double-buffered, so ONE
      // producer barrier per tile suffices for the dense / stem modes; the deformable sample table is a single
      // buffer and needs the extra barrier before it is overwritten.
      long long* rowinfo = rowbase + (tile_it & 1) * TC_BM;
      if (DEFORM) named_bar<1, TC_PRODUCERS>();   // every producer is done with the previous tile's sample table
      for (int r = pt; r < TC_BM; r += TC_PRODUCERS) {
        const long long pg = tile_pixel(mt, r);
        long long v = -1;
        if (pg >= 0) {
          const int n = (int)(pg / HoWo), pp = (int)(pg - (long long)n * HoWo);
          const int ho = pp / p.Wo, wo = pp - ho * p.Wo;
          if (DEFORM) v = (long long)n * p.H * p.W * (long long)p.Cin * (XPAIR ? 2 : 1);
          else v = ((long long)n << 40) | ((long long)(ho * p.sh - p.ph + (1 << 19)) << 20) | (long long)(wo * p.sw - p.pw + (1 << 19));
        }
        rowinfo[r] = v;
      }
      // deformable: per-tile sample table (channel independent), one entry per (tap, pixel)
      for (int e = pt; e < (DEFORM ? KHW * TC_BM : 0); e += TC_PRODUCERS) {
        const int tap = e / TC_BM, r = e - tap * TC_BM;
        const long long pg = tile_pixel(mt, r);
        const int ki = tap / p.kw, kj = tap - ki * p.kw;
        {
          float4 wv = make_float4(0.f, 0.f, 0.f, 0.f);
          int4 ov = make_int4(0, 0, 0, 0);
          if (pg >= 0) {
            const int n = (int)(pg / HoWo), pp = (int)(pg - (long long)n * HoWo);
            const int ho = pp / p.Wo, wo = pp - ho * p.Wo;
            const float* offp = p.offset + ((size_t)n * 2 * KHW + 2 * tap) * HoWo + pp;
            const float oh = __ldg(offp), ow = __ldg(offp + HoWo);
            const float h = (float)(ho * p.sh - p.ph + ki * p.dh) + oh;
            const float w = (float)(wo * p.sw - p.pw + kj * p.dw) + ow;
            if (h > -1.f && w > -1.f && h < (float)p.H && w < (float)p.W) {  // deform_conv_kernel.cu:229
              const int hl = (int)floorf(h), wl = (int)floorf(w), hh = hl + 1, wh = wl + 1;
              const float lh = h - hl, lw = w - wl, ch = 1.f - lh, cw = 1.f - lw;
              const bool t_ok = hl >= 0, b_ok = hh <= p.H - 1, l_ok = wl >= 0, r_ok = wh <= p.W - 1;
              float m = 1.f;
              if (p.mask) m = __ldg(p.mask + ((size_t)n * KHW + tap) * HoWo + pp);
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
          if (XPAIR) {   // pair gather: element offsets in the 2*Cin-channel tensor, fp32 weights
            ov.x *= 2 * p.Cin; ov.y *= 2 * p.Cin; ov.z *= 2 * p.Cin; ov.w *= 2 * p.Cin;
            tw[e] = wv;
          } else if (XBF16) {   // bf16 gather blends in packed bf16x2: weights replicated into both halves, offsets in elements
            ov.x *= p.Cin; ov.y *= p.Cin; ov.z *= p.Cin; ov.w *= p.Cin;
            uint4 wp;
            wp.x = pack_bf16x2(wv.x, wv.x); wp.y = pack_bf16x2(wv.y, wv.y);
            wp.z = pack_bf16x2(wv.z, wv.z); wp.w = pack_bf16x2(wv.w, wv.w);
            reinterpret_cast<uint4*>(tw)[e] = wp;
          } else {
            tw[e] = wv;
          }
          to[e] = ov;
        }
      }
      named_bar<1, TC_PRODUCERS>();   // row info (and sample table) visible to all producers
      ++tile_it;

      for (int kb = (int)((uint32_t)(group - (int)g0) & 1u); kb < num_kb; kb += TC_GROUPS) {  // ring parity == group
        const uint32_t g = g0 + (uint32_t)kb;
        const uint32_t s = g % (uint32_t)p.stages, it = g / (uint32_t)p.stages;
        mbar_wait(bar_empty + 8 * s, (it & 1u) ^ 1u);
        uint8_t* stage = sm + L.stages + (size_t)s * L.stage_bytes;
        uint8_t* a_hi = stage;
        uint8_t* b_hi = stage + L.a_bytes;
        uint8_t* a_lo = stage + L.a_bytes + L.b_bytes;
        uint8_t* b_lo = a_lo + L.a_bytes;
        // k-block order: dense = tap-major (matches the packed weight columns); deformable = CHANNEL-CHUNK-major, so
        // that the nine taps x four bilinear corners of one 64-channel chunk -- which revisit the same few hundred
        // 128-byte lines of the input -- run back to back and hit in L1 instead of going to L2 36 times.
        const int tap = DEFORM ? kb % KHW : kb / cchunks;
        const int cck = DEFORM ? kb / KHW : kb - tap * cchunks;
        const int c0 = cck * TC_BK + j * 8;
        const size_t kcol = (size_t)tap * p.Cin + (size_t)cck * TC_BK;   // == kb * 64 for the dense modes
        const int tki = tap / p.kw, tdy = tki * p.dh, tdx = (tap - tki * p.kw) * p.dw;   // dense: tap displacement
        // ---- B: BN rows x 8 chunks of packed bf16 weights, cp.async straight into the swizzled stage
        //      (no registers, overlaps the A gather below) ----
        for (int r = r_first; r < p.BN; r += 32) {
          const size_t gi = (size_t)(n0 + r) * Kp + (SMALLC ? (size_t)kb * TC_BK : kcol) + j * 8;
          const uint32_t soff = (uint32_t)r * 128u + (uint32_t)((j ^ (r & 7)) << 4);
          cp_async16(smem_u32(b_hi + soff), p.w_hi + gi);
          if (x3) cp_async16(smem_u32(b_lo + soff), p.w_lo + gi);
        }
        cp_async_commit();
        // ---- A: gather 128 rows x 8 chunks ----
        if (SMALLC) {
          // tiny Cin (stem): every k of the flattened (ky,kx,c) axis is an independent scalar read of the NCHW image
          const float* xf = reinterpret_cast<const float*>(p.x);
#pragma unroll 1
          for (int pass = 0; pass < TC_BM / 32; ++pass) {
            const int r = r_first + pass * 32;
            const long long rb = rowinfo[r];
            float v[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) v[q] = 0.f;
            if (rb >= 0) {
              const int n = (int)(rb >> 40), h0 = (int)((rb >> 20) & 0xfffff) - (1 << 19), w0 = (int)(rb & 0xfffff) - (1 << 19);
              const float* xn = xf + (size_t)n * p.Cin * p.H * p.W;
#pragma unroll
              for (int q = 0; q < 8; ++q) {
                const int e = ti[kb * TC_BK + j * 8 + q];
                if (e >= 0) {
                  const int hi = h0 + (e >> 16), wi = w0 + ((e >> 8) & 0xff), c = e & 0xff;
                  if (hi >= 0 && hi < p.H && wi >= 0 && wi < p.W) v[q] = __ldg(xn + ((size_t)c * p.H + hi) * p.W + wi);
                }
              }
            }
            const uint32_t soff = (uint32_t)r * 128u + (uint32_t)((j ^ (r & 7)) << 4);
            const uint4 hi4 = pack_bf16x8(v);
            *reinterpret_cast<uint4*>(a_hi + soff) = hi4;
            if (x3) *reinterpret_cast<uint4*>(a_lo + soff) = pair_lo8(v, hi4);
          }
        } else if (!DEFORM && XPAIR) {
          // dense, hi/lo pair activations: the hi and lo 128-byte rows ARE the smem rows of the two A tiles -> two cp.async
          // of 16 B per (row, chunk) straight into the swizzled stage (zero-fill for padding / out-of-range rows)
          const __nv_bfloat16* xh = reinterpret_cast<const __nv_bfloat16*>(p.x);
#pragma unroll
          for (int pass = 0; pass < TC_BM / 32; ++pass) {
            const int r = r_first + pass * 32;
            const long long rb = rowinfo[r];
            const int hi = (int)((rb >> 20) & 0xfffff) - (1 << 19) + tdy, wi = (int)(rb & 0xfffff) - (1 << 19) + tdx;
            const bool ok = rb >= 0 && hi >= 0 && hi < p.H && wi >= 0 && wi < p.W;
            const __nv_bfloat16* src = ok ? xh + (((size_t)(rb >> 40) * p.H + hi) * p.W + wi) * (size_t)(2 * p.Cin) + c0 : xh;
            const uint32_t soff = (uint32_t)r * 128u + (uint32_t)((j ^ (r & 7)) << 4);
            cp_async16_zfill(smem_u32(a_hi + soff), src, ok ? 16u : 0u);
            cp_async16_zfill(smem_u32(a_lo + soff), ok ? src + p.Cin : xh, ok ? 16u : 0u);
          }
        } else if (DEFORM && XPAIR) {
          // deformable, hi/lo pair activations: 8 lanes x 16 B cover a row's 64 channels of one plane; per corner one hi and
          // one lo load, blended and split again by pair_blend8 (pair.cuh), the blend of the window kernel (dcn_win.cu).
          const __nv_bfloat16* xh = reinterpret_cast<const __nv_bfloat16*>(p.x);
#pragma unroll 1
          for (int pass = 0; pass < TC_BM / 32; ++pass) {
            const int r = r_first + pass * 32;
            const long long rb = rowinfo[r];
            uint4 hi = make_uint4(0u, 0u, 0u, 0u), lo = hi;
            if (rb >= 0) {
              const __nv_bfloat16* xb = xh + rb + c0;
              const float4 wv = tw[tap * TC_BM + r];
              const int4 ov = to[tap * TC_BM + r];
              const uint4 ha = __ldg(reinterpret_cast<const uint4*>(xb + ov.x)), la = __ldg(reinterpret_cast<const uint4*>(xb + ov.x + p.Cin));
              const uint4 hb = __ldg(reinterpret_cast<const uint4*>(xb + ov.y)), lb = __ldg(reinterpret_cast<const uint4*>(xb + ov.y + p.Cin));
              const uint4 hd = __ldg(reinterpret_cast<const uint4*>(xb + ov.z)), ld = __ldg(reinterpret_cast<const uint4*>(xb + ov.z + p.Cin));
              const uint4 he = __ldg(reinterpret_cast<const uint4*>(xb + ov.w)), le = __ldg(reinterpret_cast<const uint4*>(xb + ov.w + p.Cin));
              const uint4 hc[4] = {ha, hb, hd, he}, lc[4] = {la, lb, ld, le};
              pair_blend8(wv, hc, lc, hi, lo);
            }
            const uint32_t soff = (uint32_t)r * 128u + (uint32_t)((j ^ (r & 7)) << 4);
            *reinterpret_cast<uint4*>(a_hi + soff) = hi;
            *reinterpret_cast<uint4*>(a_lo + soff) = lo;
          }
        } else if (!DEFORM && XBF16) {
          // dense, bf16 activations: the 128-byte row IS the smem row -> cp.async 16 B per (row, chunk)
          // straight into the swizzled stage (zero-fill for padding / out-of-range rows), no registers.
          const __nv_bfloat16* xh = reinterpret_cast<const __nv_bfloat16*>(p.x);
#pragma unroll
          for (int pass = 0; pass < TC_BM / 32; ++pass) {
            const int r = r_first + pass * 32;
            const long long rb = rowinfo[r];
            const int hi = (int)((rb >> 20) & 0xfffff) - (1 << 19) + tdy, wi = (int)(rb & 0xfffff) - (1 << 19) + tdx;
            const bool ok = rb >= 0 && hi >= 0 && hi < p.H && wi >= 0 && wi < p.W;
            const __nv_bfloat16* src = ok ? xh + (((size_t)(rb >> 40) * p.H + hi) * p.W + wi) * p.Cin + c0 : xh;
            const uint32_t soff = (uint32_t)r * 128u + (uint32_t)((j ^ (r & 7)) << 4);
            cp_async16_zfill(smem_u32(a_hi + soff), src, ok ? 16u : 0u);
          }
        } else if (!DEFORM) {
          const float* xf = reinterpret_cast<const float*>(p.x);
          // dense: a row's 64 fp32 channels (256 B) are read by 16 consecutive lanes, 16 B each, so every
          // warp-wide LDG.128 covers two fully used 256-byte spans; all eight loads of a thread are
          // issued before the first conversion (memory-level parallelism); each lane then stores 4 bf16
          // (8 B) into its half of the swizzled 16-byte chunk.
          const int l16 = gt & 15;            // 4-channel group inside the 64-channel row
          const int rr0 = gt >> 4;            // 16 rows per pass
          const int cg = c0 - j * 8 + l16 * 4;  // first channel of this lane's group
          float4 qv[TC_BM / 16];
#pragma unroll
          for (int pass = 0; pass < TC_BM / 16; ++pass) {
            const int r = rr0 + pass * 16;
            const long long rb = rowinfo[r];
            const int hi = (int)((rb >> 20) & 0xfffff) - (1 << 19) + tdy, wi = (int)(rb & 0xfffff) - (1 << 19) + tdx;
            qv[pass] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (rb >= 0 && hi >= 0 && hi < p.H && wi >= 0 && wi < p.W)
              qv[pass] = __ldg(reinterpret_cast<const float4*>(xf + (((size_t)(rb >> 40) * p.H + hi) * p.W + wi) * p.Cin + cg));
          }
#pragma unroll
          for (int pass = 0; pass < TC_BM / 16; ++pass) {
            const int r = rr0 + pass * 16;
            const uint32_t soff = (uint32_t)r * 128u + (uint32_t)(((l16 >> 1) ^ (r & 7)) << 4) + (uint32_t)((l16 & 1) << 3);
            const float4 v = qv[pass];
            const uint2 hi = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
            *reinterpret_cast<uint2*>(a_hi + soff) = hi;
            if (x3) *reinterpret_cast<uint2*>(a_lo + soff) = make_uint2(pair_lo2(v.x, v.y, hi.x), pair_lo2(v.z, v.w, hi.y));
          }
        } else if (XBF16) {
          // deformable, bf16 activations: 4 lanes x 32 B cover a row's 64 channels (two 16-byte loads per corner,
          // one address computation); the four corners are blended in packed bf16x2 (HFMA2.BF16: 4 ops per 8
          // channels and corner pair instead of 8 unpack + 8 FMA + pack) with the tile's sample table, whose
          // weights are stored as replicated bf16 pairs.  This kernel is issue-bound, so instructions per gathered
          // element are what matters.
          const __nv_bfloat16* xh = reinterpret_cast<const __nv_bfloat16*>(p.x);
          const int j2 = gt & 3, rr0 = gt >> 2;              // 64 rows per pass
          const int cp0 = c0 - j * 8 + j2 * 16;              // first channel of this lane's 16-channel slice
          const uint4* twp = reinterpret_cast<const uint4*>(tw);
#pragma unroll 1
          for (int pass = 0; pass < TC_BM / 64; ++pass) {
            const int r = rr0 + pass * 64;
            const long long rb = rowinfo[r];
            uint4 o0 = make_uint4(0u, 0u, 0u, 0u), o1 = o0;
            if (rb >= 0) {
              const __nv_bfloat16* xb = xh + rb + cp0;
              const uint4 wv = twp[tap * TC_BM + r];
              const int4 ov = to[tap * TC_BM + r];
              // 32 bytes per corner (two 16-byte loads): 4 lanes cover a row's full 128-byte line, so the L1
              // wavefront count stays that of the 8-lane x 16-byte mapping while the address work is halved
              uint4 a0, a1, b0, b1, d0, d1, e0, e1;
              ldg256(xb + ov.x, a0, a1);
              ldg256(xb + ov.y, b0, b1);
              ldg256(xb + ov.z, d0, d1);
              ldg256(xb + ov.w, e0, e1);
              o0.x = bf2_blend(wv, a0.x, b0.x, d0.x, e0.x); o0.y = bf2_blend(wv, a0.y, b0.y, d0.y, e0.y);
              o0.z = bf2_blend(wv, a0.z, b0.z, d0.z, e0.z); o0.w = bf2_blend(wv, a0.w, b0.w, d0.w, e0.w);
              o1.x = bf2_blend(wv, a1.x, b1.x, d1.x, e1.x); o1.y = bf2_blend(wv, a1.y, b1.y, d1.y, e1.y);
              o1.z = bf2_blend(wv, a1.z, b1.z, d1.z, e1.z); o1.w = bf2_blend(wv, a1.w, b1.w, d1.w, e1.w);
            }
            const uint32_t rbase = (uint32_t)r * 128u, rx = (uint32_t)(r & 7);
            *reinterpret_cast<uint4*>(a_hi + rbase + ((((uint32_t)j2 * 2u) ^ rx) << 4)) = o0;
            *reinterpret_cast<uint4*>(a_hi + rbase + ((((uint32_t)j2 * 2u + 1u) ^ rx) << 4)) = o1;
          }
        } else {
          const float* xf = reinterpret_cast<const float*>(p.x);
          // deformable: same coalesced lane mapping; per (row, 4-channel group) four 16-byte corner reads,
          // blended in fp32 with the tile's sample table (weights already carry validity and the v2 mask).
          const int l16 = gt & 15;
          const int rr0 = gt >> 4;
          const int cg = c0 - j * 8 + l16 * 4;
#pragma unroll 2
          for (int pass = 0; pass < TC_BM / 16; ++pass) {
            const int r = rr0 + pass * 16;
            const long long rb = rowinfo[r];
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (rb >= 0) {
              const float* xb = xf + rb + cg;
              const float4 wv = tw[tap * TC_BM + r];
              const int4 ov = to[tap * TC_BM + r];
              const float4 a0 = __ldg(reinterpret_cast<const float4*>(xb + (size_t)ov.x * p.Cin));
              const float4 b0 = __ldg(reinterpret_cast<const float4*>(xb + (size_t)ov.y * p.Cin));
              const float4 d0 = __ldg(reinterpret_cast<const float4*>(xb + (size_t)ov.z * p.Cin));
              const float4 e0 = __ldg(reinterpret_cast<const float4*>(xb + (size_t)ov.w * p.Cin));
              v.x = wv.x * a0.x + wv.y * b0.x + wv.z * d0.x + wv.w * e0.x;
              v.y = wv.x * a0.y + wv.y * b0.y + wv.z * d0.y + wv.w * e0.y;
              v.z = wv.x * a0.z + wv.y * b0.z + wv.z * d0.z + wv.w * e0.z;
              v.w = wv.x * a0.w + wv.y * b0.w + wv.z * d0.w + wv.w * e0.w;
            }
            const uint32_t soff = (uint32_t)r * 128u + (uint32_t)(((l16 >> 1) ^ (r & 7)) << 4) + (uint32_t)((l16 & 1) << 3);
            const uint2 hi = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
            *reinterpret_cast<uint2*>(a_hi + soff) = hi;
            if (x3) *reinterpret_cast<uint2*>(a_lo + soff) = make_uint2(pair_lo2(v.x, v.y, hi.x), pair_lo2(v.z, v.w, hi.y));
          }
        }
        cp_async_commit();
        if (deferred) {
          if (pend_s >= 0) {
            cp_async_wait_but2();   // everything except this k-block's two commit groups has landed
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_full + 8 * pend_s);
          }
          pend_s = (int)s;
        } else {
          cp_async_wait_all();
          fence_proxy_async();  // generic-proxy stores -> visible to the tensor core (async proxy)
          __syncwarp();
          if (lane == 0) mbar_arrive(bar_full + 8 * s);
        }
      }
      g0 += (uint32_t)num_kb;
    }
    if (pend_s >= 0) {
      cp_async_wait_all();
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_full + 8 * pend_s);
    }
  } else {
    // =============================== CONSUMERS (warps 0-3) ===============================
    const uint32_t dhi = wg_desc_hi(1024);          // 8-row groups of 128-byte rows
    const bool vec_ptrs_ok = (((uintptr_t)p.y) & 15) == 0 && (!p.residual || (((uintptr_t)p.residual) & 15) == 0);
    float* stf = reinterpret_cast<float*>(sm + L.epi);
    float d0[BN / 2], d1[BN / 2];                   // tile rows [0, 64) and [64, 128)
    uint32_t s = 0, ph = 0;
    for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const long long mt = tile / n_tiles;
      const int n0 = (int)(tile % n_tiles) * BN;
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(bar_full + 8 * s, ph);
        const uint32_t st0 = base + L.stages + s * L.stage_bytes;
        const uint32_t a_hi = wg_desc_lo(st0), b_hi = wg_desc_lo(st0 + L.a_bytes);
        const uint32_t a_lo = wg_desc_lo(st0 + L.a_bytes + L.b_bytes), b_lo = wg_desc_lo(st0 + 2 * L.a_bytes + L.b_bytes);
        constexpr uint32_t h16 = 64u * 128u / 16u;      // rows 64-127: 64 rows of 128 bytes further
        wgmma_fence();
#pragma unroll
        for (uint32_t k = 0; k < TC_BK / 16; ++k) {       // 16 bf16 = 32 bytes = 2 descriptor units
          const uint32_t acc = (kb | k) ? 1u : 0u;
          const uint64_t bh = wg_desc(b_hi + 2 * k, dhi);
          if (x3) {
            const uint64_t bl = wg_desc(b_lo + 2 * k, dhi);
            Wgmma<BN>::mma(d0, wg_desc(a_lo + 2 * k, dhi), bh, acc);
            Wgmma<BN>::mma(d1, wg_desc(a_lo + h16 + 2 * k, dhi), bh, acc);
            Wgmma<BN>::mma(d0, wg_desc(a_hi + 2 * k, dhi), bl, 1u);
            Wgmma<BN>::mma(d1, wg_desc(a_hi + h16 + 2 * k, dhi), bl, 1u);
            Wgmma<BN>::mma(d0, wg_desc(a_hi + 2 * k, dhi), bh, 1u);
            Wgmma<BN>::mma(d1, wg_desc(a_hi + h16 + 2 * k, dhi), bh, 1u);
          } else {
            Wgmma<BN>::mma(d0, wg_desc(a_hi + 2 * k, dhi), bh, acc);
            Wgmma<BN>::mma(d1, wg_desc(a_hi + h16 + 2 * k, dhi), bh, acc);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();                                // the previous k-block's wgmmas have read their stage
        wgmma_fence_acc(d0);
        wgmma_fence_acc(d1);
        if (prev >= 0 && lane == 0) mbar_arrive(bar_empty + 8 * prev);
        prev = (int)s;
        if (++s == (uint32_t)p.stages) { s = 0; ph ^= 1u; }
      }
      wgmma_wait<0>();
      wgmma_fence_acc(d0);
      wgmma_fence_acc(d1);
      if (prev >= 0 && lane == 0) mbar_arrive(bar_empty + 8 * prev);

      // ---- epilogue: 32 accumulator columns at a time through shared memory, thread = tile row ----
      const int q = warp;
      const int m = q * 32 + lane;
      const long long pg = tile_pixel(mt, m);
      const bool row_ok = pg >= 0;
      const int n_img = row_ok ? (int)(pg / HoWo) : 0;
      const int pp = row_ok ? (int)(pg - (long long)n_img * HoWo) : 0;
      const uint32_t trow = smem_u32(stf + (size_t)m * TC_EPI_PITCH);
      for (int cb = 0; cb < BN; cb += 32) {
        if (n0 + cb >= p.Cout) break;                   // zero-padded weight rows beyond Cout (CTA-uniform)
        named_bar(2, TC_CONSUMERS);                     // the previous chunk has been read
#pragma unroll
        for (int c = 0; c < BN; c += 32)
          if (c == cb) {
            acc_stage<BN, 32>(d0, stf, TC_EPI_PITCH, 0, c);
            acc_stage<BN, 32>(d1, stf, TC_EPI_PITCH, 64, c);
          }
        named_bar(2, TC_CONSUMERS);
        if (p.out_nhwc && (p.Cout & 7) == 0 && vec_ptrs_ok) {
          // ---- NHWC: this warp's 32 staged rows x 32 columns (+bias, in place) are written out row-wise: 4 (bf16) or
          //      8 (fp32) lanes cover one row's 64 / 128 contiguous bytes, so every store -- and every residual read -- is
          //      made of fully used 32-byte sectors instead of one 16-byte fragment per 512-byte-strided row. ----
          float* st = stf + (size_t)q * 32 * TC_EPI_PITCH;
          const bool y16 = p.y_bf16 || p.y_pair;          // 16-bit storage: 8 columns (16 B) per lane
          const size_t ypitch = p.y_pair ? 2 * (size_t)p.Cout : (size_t)p.Cout;   // elements per stored pixel
          const int lpr = y16 ? 4 : 8;                    // lanes per row in the write-out phase
          const int rpi = 32 / lpr;                       // rows per iteration
          const int sub = lane % lpr, rsub = lane / lpr;
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            uint32_t rr[16];
            acc_ld16(trow + (uint32_t)(c * 16) * 4u, rr);
            const int co0 = n0 + cb + c * 16;
            float4* dst = reinterpret_cast<float4*>(st + lane * TC_EPI_PITCH + c * 16);
#pragma unroll
            for (int g4 = 0; g4 < 4; ++g4) {
              float4 o = make_float4(__uint_as_float(rr[g4 * 4]), __uint_as_float(rr[g4 * 4 + 1]),
                                     __uint_as_float(rr[g4 * 4 + 2]), __uint_as_float(rr[g4 * 4 + 3]));
              if (p.bias && co0 + g4 * 4 + 3 < p.Cout) {
                o.x += __ldg(p.bias + co0 + g4 * 4); o.y += __ldg(p.bias + co0 + g4 * 4 + 1);
                o.z += __ldg(p.bias + co0 + g4 * 4 + 2); o.w += __ldg(p.bias + co0 + g4 * 4 + 3);
              }
              dst[g4] = o;
            }
          }
          __syncwarp();
          const int ce = y16 ? sub * 8 : sub * 4;        // first staged column of this lane
          const int co = n0 + cb + ce;
          if (co < p.Cout) {
            for (int it = 0; it < lpr; ++it) {
              const int row = it * rpi + rsub;
              const long long pgr = tile_pixel(mt, q * 32 + row);
              if (pgr < 0) continue;
              size_t ridx = (size_t)pgr * ypitch + co;
              if (p.residual && p.res_up2) {
                const int ni = (int)(pgr / HoWo), ppr = (int)(pgr - (long long)ni * HoWo);
                const int ho = ppr / p.Wo, wo = ppr - ho * p.Wo;
                ridx = (((size_t)ni * (p.Ho >> 1) + (ho >> 1)) * (p.Wo >> 1) + (wo >> 1)) * ypitch + co;
              }
              const float* src = st + row * TC_EPI_PITCH + ce;
              if (p.y_pair) {
                // hi/lo pair output: residual = hi + lo (exact in fp32), result split into bf16(o) and bf16(o - hi)
                const float4 a = *reinterpret_cast<const float4*>(src), b = *reinterpret_cast<const float4*>(src + 4);
                float o[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
                if (p.residual) {
                  const __nv_bfloat16* rp = reinterpret_cast<const __nv_bfloat16*>(p.residual) + ridx;
                  const uint4 rh = __ldg(reinterpret_cast<const uint4*>(rp)), rl = __ldg(reinterpret_cast<const uint4*>(rp + p.Cout));
                  const uint32_t hw[4] = {rh.x, rh.y, rh.z, rh.w}, lw[4] = {rl.x, rl.y, rl.z, rl.w};
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    o[2 * e] += pair_x(hw[e], lw[e]);
                    o[2 * e + 1] += pair_y(hw[e], lw[e]);
                  }
                }
                if (p.relu) {
#pragma unroll
                  for (int e = 0; e < 8; ++e) o[e] = fmaxf(o[e], 0.f);
                }
                uint4 hi, lo;
                split_pair8(o, hi, lo);
                __nv_bfloat16* yp = reinterpret_cast<__nv_bfloat16*>(p.y) + (size_t)pgr * ypitch + co;
                *reinterpret_cast<uint4*>(yp) = hi;
                *reinterpret_cast<uint4*>(yp + p.Cout) = lo;
              } else if (p.y_bf16) {
                const float4 a = *reinterpret_cast<const float4*>(src), b = *reinterpret_cast<const float4*>(src + 4);
                float o[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
                if (p.residual) {
                  const uint4 rv = __ldg(reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.residual) + ridx));
                  const uint32_t rw[4] = {rv.x, rv.y, rv.z, rv.w};
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    o[2 * e] += bf16x2_x(rw[e]);
                    o[2 * e + 1] += bf16x2_y(rw[e]);
                  }
                }
                if (p.relu) {
#pragma unroll
                  for (int e = 0; e < 8; ++e) o[e] = fmaxf(o[e], 0.f);
                }
                *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.y) + (size_t)pgr * p.Cout + co) = pack_bf16x8(o);
              } else {
                float4 o = *reinterpret_cast<const float4*>(src);
                if (p.residual) {
                  const float4 rv = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.residual) + ridx));
                  o.x += rv.x; o.y += rv.y; o.z += rv.z; o.w += rv.w;
                }
                if (p.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
                *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.y) + (size_t)pgr * p.Cout + co) = o;
              }
            }
          }
          continue;
        }
        // ---- per-lane path (NCHW outputs, odd channel counts) ----
        for (int col = cb; col < cb + 32; col += 16) {
          uint32_t rr[16];
          acc_ld16(trow + (uint32_t)(col - cb) * 4u, rr);
          if (!row_ok) continue;
          const int co0 = n0 + col;
          if (co0 >= p.Cout) continue;
          float o16[16];
#pragma unroll
          for (int e = 0; e < 16; ++e) o16[e] = __uint_as_float(rr[e]);
          if (p.bias) {
#pragma unroll
            for (int e = 0; e < 16; ++e) if (co0 + e < p.Cout) o16[e] += __ldg(p.bias + co0 + e);
          }
          if (p.out_nhwc) {
            const size_t oidx = (size_t)pg * p.Cout + co0;
            // FPN top-down path (models/fpn.py:88-93): lateral conv + nearest-2x-upsampled coarser map, fused:
            // the residual is indexed at (ho/2, wo/2) of the half-resolution tensor instead of being materialised.
            size_t ridx = oidx;
            if (p.res_up2) {
              const int ho = pp / p.Wo, wo = pp - ho * p.Wo;
              ridx = (((size_t)n_img * (p.Ho >> 1) + (ho >> 1)) * (p.Wo >> 1) + (wo >> 1)) * p.Cout + co0;
            }
            const bool full = (co0 + 15 < p.Cout) && ((p.Cout & 7) == 0) && vec_ptrs_ok;
            if (p.y_bf16) {
              __nv_bfloat16* yo = reinterpret_cast<__nv_bfloat16*>(p.y) + oidx;
              const __nv_bfloat16* ro = p.residual ? reinterpret_cast<const __nv_bfloat16*>(p.residual) + ridx : nullptr;
              if (full) {
                if (ro) {
                  const uint4 r0 = __ldg(reinterpret_cast<const uint4*>(ro)), r1 = __ldg(reinterpret_cast<const uint4*>(ro) + 1);
                  const uint32_t rw[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
                  for (int q = 0; q < 8; ++q) {
                    o16[2 * q] += bf16x2_x(rw[q]);
                    o16[2 * q + 1] += bf16x2_y(rw[q]);
                  }
                }
                if (p.relu) {
#pragma unroll
                  for (int e = 0; e < 16; ++e) o16[e] = fmaxf(o16[e], 0.f);
                }
                reinterpret_cast<uint4*>(yo)[0] = pack_bf16x8(o16);
                reinterpret_cast<uint4*>(yo)[1] = pack_bf16x8(o16 + 8);
              } else {
#pragma unroll
                for (int e = 0; e < 16; ++e) {
                  if (co0 + e >= p.Cout) break;
                  float o = o16[e];
                  if (ro) o += __bfloat162float(ro[e]);
                  if (p.relu) o = fmaxf(o, 0.f);
                  yo[e] = __float2bfloat16_rn(o);
                }
              }
            } else {
              float* yo = reinterpret_cast<float*>(p.y) + oidx;
              const float* ro = p.residual ? reinterpret_cast<const float*>(p.residual) + ridx : nullptr;
              if (full) {
#pragma unroll
                for (int g4 = 0; g4 < 4; ++g4) {
                  float4 o = make_float4(o16[g4 * 4], o16[g4 * 4 + 1], o16[g4 * 4 + 2], o16[g4 * 4 + 3]);
                  if (ro) {
                    const float4 rv = __ldg(reinterpret_cast<const float4*>(ro + g4 * 4));
                    o.x += rv.x; o.y += rv.y; o.z += rv.z; o.w += rv.w;
                  }
                  if (p.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
                  *reinterpret_cast<float4*>(yo + g4 * 4) = o;
                }
              } else {
#pragma unroll
                for (int e = 0; e < 16; ++e) {
                  if (co0 + e >= p.Cout) break;
                  float o = o16[e];
                  if (ro) o += __ldg(ro + e);
                  if (p.relu) o = fmaxf(o, 0.f);
                  yo[e] = o;
                }
              }
            }
          } else {  // NCHW: for a fixed cout the 32 lanes of a warp write 32 consecutive pixels
#pragma unroll
            for (int e = 0; e < 16; ++e) {
              const int co = co0 + e;
              if (co >= p.Cout) break;
              const size_t oidx = ((size_t)n_img * p.Cout + co) * HoWo + pp;
              float o = o16[e];
              if (p.y_bf16) {
                if (p.residual) o += __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.residual)[oidx]);
                if (p.relu) o = fmaxf(o, 0.f);
                reinterpret_cast<__nv_bfloat16*>(p.y)[oidx] = __float2bfloat16_rn(o);
              } else {
                if (p.residual) o += __ldg(reinterpret_cast<const float*>(p.residual) + oidx);
                if (p.relu) o = fmaxf(o, 0.f);
                if (p.sig_from >= 0 && co >= p.sig_from) o = 1.f / (1.f + expf(-o));
                reinterpret_cast<float*>(p.y)[oidx] = o;
              }
            }
          }
        }
      }
    }
  }
}

// ----------------------------------------------------------------------------------------------
// weight pre-pack: fp32 [Cout,Cin,kh,kw] -> bf16 hi / lo planes [Cout_pad][KHW*Cin], k = tap*Cin + c
// ----------------------------------------------------------------------------------------------
__global__ void pack_weight_kernel(const float* __restrict__ w, int Cout, int Cin, int KHW, int Cout_pad, int Kp,
                                   uint16_t* __restrict__ hi, uint16_t* __restrict__ lo) {
  const size_t total = (size_t)Cout_pad * Kp;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int kk = (int)(i % (size_t)Kp);
    const int co = (int)(i / (size_t)Kp);
    const int tap = kk / Cin, c = kk - tap * Cin;
    const float v = (co < Cout && kk < KHW * Cin) ? w[((size_t)co * Cin + c) * KHW + tap] : 0.f;
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    hi[i] = *reinterpret_cast<const uint16_t*>(&h);
    lo[i] = *reinterpret_cast<const uint16_t*>(&l);
  }
}

static int tc_kp(int Cin, int KHW) { return (KHW * Cin + TC_BK - 1) / TC_BK * TC_BK; }

size_t tc_packed_weight_bytes(int Cout, int Cin, int kh, int kw) {
  return (size_t)2 * cout_pad(Cout) * tc_kp(Cin, kh * kw) * sizeof(uint16_t);
}

int tc_pack_weight(const float* w, int Cout, int Cin, int kh, int kw, void* packed, cudaStream_t stream) {
  const int Cout_pad = cout_pad(Cout), KHW = kh * kw, Kp = tc_kp(Cin, KHW);
  uint16_t* hi = reinterpret_cast<uint16_t*>(packed);
  uint16_t* lo = hi + (size_t)Cout_pad * Kp;
  const size_t total = (size_t)Cout_pad * Kp;
  int blocks = (int)((total + 255) / 256);
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  pack_weight_kernel<<<blocks, 256, 0, stream>>>(w, Cout, Cin, KHW, Cout_pad, Kp, hi, lo);
  UPS_CHECK_LAUNCH();
  return 0;
}

// Cin % 64 == 0 (NHWC gather / cp.async), or a tiny Cin <= 8 (the RGB stem: NCHW fp32 input, flattened K)
bool tc_supported(int Cin, int kh, int kw, int dg) {
  return ((Cin % TC_BK) == 0 || Cin <= 8) && dg == 1 && kh * kw <= 49 && kh <= 15 && kw <= 15;
}

template <int BN>
static cudaError_t tc_configure() {
  const void* k[] = {(const void*)igemm_tc_kernel<0, 0, BN>, (const void*)igemm_tc_kernel<0, 1, BN>, (const void*)igemm_tc_kernel<0, 2, BN>,
                     (const void*)igemm_tc_kernel<1, 0, BN>, (const void*)igemm_tc_kernel<1, 1, BN>, (const void*)igemm_tc_kernel<1, 2, BN>,
                     (const void*)igemm_tc_kernel<2, 0, BN>};
  for (const void* f : k) {
    const cudaError_t e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
  }
  // deformable instantiations: prefer the smallest shared-memory carve-out that fits, the rest of the 256 KB is L1
  for (int i = 3; i < 6; ++i) (void)cudaFuncSetAttribute(k[i], cudaFuncAttributePreferredSharedMemoryCarveout, 60);
  return cudaSuccess;
}

template <int BN>
static void tc_launch(const TcParams& p, bool deform, bool smallc, dim3 grid, size_t smem, cudaStream_t stream) {
  if (smallc) igemm_tc_kernel<2, 0, BN><<<grid, TC_THREADS, smem, stream>>>(p);
  else if (p.x_pair) {
    if (deform) igemm_tc_kernel<1, 2, BN><<<grid, TC_THREADS, smem, stream>>>(p);
    else igemm_tc_kernel<0, 2, BN><<<grid, TC_THREADS, smem, stream>>>(p);
  } else if (p.x_bf16) {
    if (deform) igemm_tc_kernel<1, 1, BN><<<grid, TC_THREADS, smem, stream>>>(p);
    else igemm_tc_kernel<0, 1, BN><<<grid, TC_THREADS, smem, stream>>>(p);
  } else {
    if (deform) igemm_tc_kernel<1, 0, BN><<<grid, TC_THREADS, smem, stream>>>(p);
    else igemm_tc_kernel<0, 0, BN><<<grid, TC_THREADS, smem, stream>>>(p);
  }
}

int launch_igemm_tc(TcParams p, const void* packed, cudaStream_t stream) {
  const int KHW = p.kh * p.kw;
  if (!tc_supported(p.Cin, p.kh, p.kw, 1)) return UPSNET_E_UNSUPPORTED;
  {  // stride-1 dense layers on bf16 NHWC activations: operands by TMA, no gather threads (igemm_tma.cu)
    const int rc = launch_igemm_tma(p, packed, stream);
    if (rc != UPSNET_E_UNSUPPORTED) return rc;
  }
  if ((((uintptr_t)p.x) & 15) || (((uintptr_t)packed) & 15) || (((uintptr_t)p.y) & 15)) return UPSNET_E_BADARG;
  p.Cout_pad = cout_pad(p.Cout);
  p.w_hi = reinterpret_cast<const uint16_t*>(packed);
  p.w_lo = p.w_hi + (size_t)p.Cout_pad * tc_kp(p.Cin, KHW);
  const bool deform = p.offset != nullptr;
  const bool smallc = (p.Cin % TC_BK) != 0;
  if (deform && (p.x_bf16 || p.x_pair) && (long long)p.H * p.W * p.Cin * (p.x_pair ? 2 : 1) >= (1ll << 31)) return UPSNET_E_UNSUPPORTED;   // int32 element offsets
  if (smallc && (deform || p.x_bf16 || p.x_pair || p.dh * (p.kh - 1) > 255 || p.dw * (p.kw - 1) > 255)) return UPSNET_E_UNSUPPORTED;
  if (p.x_pair && !p.x3) return UPSNET_E_UNSUPPORTED;          // pairs are the storage format of precision bf16x3
  if (p.sig_from >= 0 && (p.out_nhwc || p.y_bf16)) return UPSNET_E_UNSUPPORTED;   // sigmoid lives in the fp32 NCHW per-lane epilogue
  if (p.x_bf16 && !p.x_pair && p.x3) return UPSNET_E_UNSUPPORTED;   // the hi/lo split needs fp32 or pair activations
  if (p.y_pair) {
    // pair output: the staged NHWC epilogue only (16-byte vectors), plain [hi Cout][lo Cout] grouping
    if (!p.out_nhwc || (p.Cout & 7) || (p.pair_group && p.pair_group != p.Cout)) return UPSNET_E_UNSUPPORTED;
    if (p.residual && (((uintptr_t)p.residual) & 15)) return UPSNET_E_UNSUPPORTED;
  }
  // tile N: as wide as the register file allows (each gathered A tile is reused by BN couts).  20 warps leave 96 registers
  // per thread (ptxas -v: 96 used); the consumer holds two m64nBN fragments = BN floats, so BN = 64 (64 floats next to the
  // addressing, a few hundred bytes spilled) is the widest that fits -- BN = 128 would need 128 registers for the fragments.
  int BN = p.Cout_pad > 64 ? 64 : p.Cout_pad;
  {  // few output tiles (FC layers, coarse pyramid levels): narrower N tiles so that every SM gets work
    const long long mt = ((long long)p.N * p.Ho * p.Wo + TC_BM - 1) / TC_BM;
    while (BN > 64 && (BN % 32) == 0 && mt * (p.Cout_pad / BN) < kNumSMs && p.Cout_pad % (BN / 2) == 0 && ((BN / 2) % 32) == 0) BN /= 2;
  }
  p.BN = BN;
  // One persistent CTA per SM: give the smem ring everything that is left after the sample table.
  const int khw_l = smallc ? 2 : KHW;   // table region: [KHW][128] entries, or the 1 KB per-k table of the stem mode
  // deformable: a short ring leaves ~100 KB of the SM's 256 KB of L1 / shared memory to the corner gathers (see the producer)
  int stages = deform ? 3 : TC_MAX_STAGES;
  TcSmem L = tc_smem_layout(deform, khw_l, BN, stages, p.x3 != 0);
  while (stages > 2 && L.total + 1024 > 220 * 1024) { --stages; L = tc_smem_layout(deform, khw_l, BN, stages, p.x3 != 0); }
  if (L.total + 1024 > 227 * 1024) return UPSNET_E_UNSUPPORTED;
  p.stages = stages;
  const long long Ptot = (long long)p.N * p.Ho * p.Wo;
  if (Ptot <= 0) return 0;
  const int sms = num_sms();
  p.tile_w = 16; p.tile_h = 8;
  auto dtiles = [&]() { return (long long)p.N * ((p.Wo + p.tile_w - 1) / p.tile_w) * ((p.Ho + p.tile_h - 1) / p.tile_h) * (p.Cout_pad / BN); };
  if (deform) {   // few tiles (coarse pyramid levels): smaller pixel blocks -> more CTAs, proportionally less gather work each
    if (dtiles() < sms / 2) { p.tile_w = 8; p.tile_h = 8; }
    if (dtiles() < sms / 2) { p.tile_h = 4; }
  }
  const long long num_tiles = (deform ? dtiles() : ((Ptot + TC_BM - 1) / TC_BM) * (p.Cout_pad / BN));
  dim3 grid((unsigned)(num_tiles < sms ? num_tiles : sms));
  const size_t smem = L.total + 1024;
  // opt in to the full 227 KB once per device (kept out of the per-launch path: CUDA-graph capture)
  static PerDeviceOnce configured;
  if (configured.need()) {
    UPS_CUDA(tc_configure<32>());
    UPS_CUDA(tc_configure<64>());
  }
  switch (BN) {
    case 32: tc_launch<32>(p, deform, smallc, grid, smem, stream); break;
    case 64: tc_launch<64>(p, deform, smallc, grid, smem, stream); break;
    default: return UPSNET_E_UNSUPPORTED;
  }
  UPS_CHECK_LAUNCH();
  return 0;
}

}  // namespace ups
