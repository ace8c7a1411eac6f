// igemm_tma.cu -- TMA-fed wgmma implicit-GEMM convolution for sm_90a (dense, stride 1, bf16 NHWC in / out).
//
// The layers that dominate the UPSNet backbone / FPN / RPN / mask head / FC path (1x1 and 3x3, stride 1,
// Cin % 64 == 0, Cout % 64 == 0; reference: models/resnet.py, models/fpn.py, models/rcnn.py) need no gather
// arithmetic at all once the activations are NHWC bf16: a tile of output pixels is a bw x bh x bn BOX of the
// 4-D tensor (C, W, H, N), and filter tap (ki, kj) of that tile is the SAME box shifted by (kj*dil - pad,
// ki*dil - pad) with out-of-range pixels reading zero.  That is exactly one tiled-mode TMA load per k-block:
//
//   A[<=128 pixels x 64 ch]  cp.async.bulk.tensor.4d  box (64, bw, bh, bn) at (c0, w0 + kj*dw - pw, h0 + ki*dh - ph, n0)
//   B[BN couts x 64 k]       cp.async.bulk.tensor.2d  box (64, BN) of the packed weights [Cout][tap*Cin + c]
//   D[128 x BN] fp32 in registers  +=  A * B^T     wgmma m64nBNk16, two warpgroups (tile rows 0-63 / 64-127)
//   epilogue (same 8 warps): accumulators -> fp32 staging rows in smem -> thread = accumulator row: +bias (+residual
//            slab, TMA-prefetched) -> ReLU -> bf16 -> SWIZZLE_128B slab in smem -> cp.async.bulk.tensor.4d store
//            (clips the box at the borders); hi/lo pair outputs skip the staging: the same steps run on the fragments
//            and write the (hi, lo) slabs from registers
//
// Both operands land in the K-major SWIZZLE_128B layout the wgmma descriptors expect (the TMA swizzle mode and
// the smem descriptor's layout type are the same permutation), so no thread touches the operands: 2 service
// warps (TMA loads, residual loads) + 8 consumer warps per persistent CTA, one CTA per SM.
// Roofline: tensor pipe for the 3x3 layers (2*P*Cout*Cin*9 flop), HBM for the 1x1 (+residual) layers
// (x + residual + y bytes); per-SM L2->smem operand traffic is (128 + BN) * 128 B per k-block.
#include <cuda.h>   // CUtensorMap + enums only; the encoder is resolved at run time (no libcuda link dependency)
#include <cuda_bf16.h>
#include <cstdlib>

#include "common.cuh"
#include "tc_ptx.cuh"
#include "tc_params.cuh"

namespace ups {

constexpr int TM_EPI_WARPS = 8;                 // consumers: two wgmma warpgroups, then the epilogue
constexpr int TM_WARP_TMA = 8, TM_WARP_RES = 9;
constexpr int TM_THREADS = 10 * 32;
constexpr int TM_MAX_STAGES = 8;
constexpr int TM_SLAB_BYTES = 128 * 128;   // 128 rows x 64 bf16
constexpr int TM_MMA_BF16 = 0, TM_MMA_WIDE = 1;   // bf16 stream: hi*hi | pair stream: hi*[hi;lo] + lo*hi

struct TmaGeom {
  const float* bias;
  int N, Ho, Wo, Cout, Cin;
  int kw, KHW, ph, pw, dh, dw;
  int bw, bh, bn;                       // M-tile box: pixels along W, along H, images (bw*bh*bn <= 128)
  int tiles_w, tiles_h, tiles_n, n_tiles;
  // optional device-side image count (<= N): tiles whose first image is >= *n_dev are skipped (the grid stays the static
  // maximum, so a captured graph keeps its shape).  Read by every role at kernel start: the TMA producer, the residual warp
  // and the consumers must walk the same tile sequence or the mbarrier rings would never drain.
  const int* n_dev;
  int BN, stages, relu, has_res;
  int res_up2;                          // residual = half-resolution map, nearest 2x up-sampling (FPN top-down)
  // direct-store epilogue (small / odd Cout, fp32 or NCHW outputs: offset convs, RPN / score / mask-logit heads)
  int direct, y_bf16, out_nhwc;
  void* y;
  int stem;                             // stride-2 tiny-Cin stem: A boxes come from the packed / padded image (5-D map)
  int sig_from;                         // direct epilogue: channels >= sig_from get a logistic sigmoid (-1 = none)
  // PAIR mode (precision bf16x3 on the TMA kernel): activations are hi/lo bf16 PAIRS -- an NHWC tensor with 2*C channels,
  // channels [0,C) = bf16(x), [C,2C) = bf16(x - hi) -- weights are the packed hi/lo planes, every k-slice issues three
  // MMAs (lo*hi, hi*lo, hi*hi) and the epilogue splits the fp32 result into a pair again.
  int x3;
  int x_lo;                             // channel coordinate of the input's lo plane (= Cin)
  int w_lo;                             // row coordinate of the weight lo plane (= Cout_pad)
  int pg;                               // output / residual pair group G: channels stored [hi G][lo G] per group (G = Cout normally)
  int res_inplace;                      // residual slabs are TMA-loaded into the (double-buffered) output slabs and updated in place
  int opairs;                           // output slab pairs that alternate (2, or 1 when shared memory is short)
  // pair mode: the hi*hi and hi*lo products share ONE instruction -- B operand = the contiguous [W_hi ; W_lo] tile of the
  // stage (N = 2 BN <= 256), accumulated in columns [0, 2 BN); lo*hi goes to columns [0, BN); the consumers add the two
  // column groups in registers and the slab epilogue works on the fragments.  Two wgmma per K slice instead of three.
  int wide;
};

// pair tensors: channel coordinate of channel n's hi value when channels are stored [hi G][lo G] per group of G (lo = +G)
__device__ __forceinline__ int pair_chan(int n, int G) { return (n / G) * 2 * G + (n % G); }

struct TmaSmem {
  uint32_t stages, out, res, acc, a_bytes, b_bytes, stage_bytes, total;
  uint32_t a_half, b_half;                                   // pair mode: offset of the lo tile inside an A / B slot
  uint32_t oslabs, res_slab;                                 // pair mode: number of (hi, lo) output slab pairs; bytes per residual slab
};
// Accumulator staging (bf16-stream slab epilogue, direct-store epilogue): 128 rows of BN fp32 (wide mode adds its two column
// groups in registers first), no padding -- the 16-byte chunk j of row r sits at chunk j ^ (r & 7), so the row-per-lane reads
// of the epilogue are conflict-free.
template <int N, int W>   // fragment of m64nN, columns [0, W) staged
__device__ __forceinline__ void acc_stage_sw(const float (&d)[N / 2], float* buf, int row0) {
  const int t = threadIdx.x & 127, l = t & 31;
  const int r = row0 + 16 * (t >> 5) + (l >> 2);
#pragma unroll
  for (int i = 0; i < W / 8; ++i) {
    const int c = 8 * i + 2 * (l & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int rr = r + 8 * h;
      const int pc = ((((c >> 2) ^ (rr & 7))) << 2) | (c & 3);
      *reinterpret_cast<float2*>(buf + (size_t)rr * W + pc) = make_float2(d[4 * i + 2 * h], d[4 * i + 2 * h + 1]);
    }
  }
}
// 16 consecutive staged fp32 of `row` from column `col` (multiple of 4); rowaddr = shared address of the row
__device__ __forceinline__ void acc_ld16_sw(uint32_t rowaddr, int row, int col, uint32_t (&r)[16]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t a = rowaddr + ((uint32_t)(((col >> 2) + i) ^ (row & 7)) << 4);
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[4 * i]), "=r"(r[4 * i + 1]), "=r"(r[4 * i + 2]), "=r"(r[4 * i + 3]) : "r"(a));
  }
}
__host__ __device__ inline TmaSmem tma_smem_layout(int BN, int stages, bool has_res, bool direct, bool x3, bool res_up2,
                                                  bool res_inplace, int opairs) {
  TmaSmem s;
  const uint32_t mul = x3 ? 2u : 1u;
  s.a_half = 128 * 128; s.b_half = (uint32_t)BN * 128;
  s.a_bytes = s.a_half * mul;
  s.b_bytes = s.b_half * mul;
  s.stage_bytes = s.a_bytes + s.b_bytes;
  s.stages = 1024;                                           // barriers live in the first KB
  s.out = s.stages + s.stage_bytes * (uint32_t)stages;
  s.res_slab = (x3 && res_up2) ? 4096u : (uint32_t)TM_SLAB_BYTES;
  if (x3) {
    // pair mode: the eight epilogue warps work on ONE 64-channel slab pair at a time (two pairs alternate so that a TMA
    // store can still be reading the first while the second is written); in-place residual: one pair per slab and buffer
    s.oslabs = direct ? 0u : (res_inplace ? 2u * (uint32_t)(BN / 64) : (uint32_t)opairs);
    s.res = s.out + s.oslabs * 2u * TM_SLAB_BYTES;
    s.acc = s.res + ((has_res && !res_inplace) ? 2u * (uint32_t)(BN / 64) * 2u * s.res_slab : 0u);
  } else {
    s.oslabs = 0;
    const uint32_t out_slabs = direct ? 0 : (BN == 64 ? 1 : 2);   // one output slab per epilogue group (TMA-store epilogue only)
    s.res = s.out + out_slabs * TM_SLAB_BYTES;
    s.acc = s.res + (has_res ? 2u * (uint32_t)(BN / 64) * TM_SLAB_BYTES : 0u);   // two residual buffers (prefetch)
  }
  // the pair slab epilogue writes the slabs straight from the fragments: no staging rows
  s.total = s.acc + ((x3 && !direct) ? 0u : 128u * (uint32_t)BN * 4u);
  return s;
}

// Roles (10 warps): warps 0-7 consumers -- two wgmma warpgroups (tile rows [64 wg, 64 wg + 64)), then the epilogue
// (pair slabs: on the fragments; staged epilogues: thread = accumulator row q * 32 + lane with q = warp & 3, column
// half = warp >> 2); warp 8 TMA operand loads, warp 9 residual-slab loads.
// Barriers: full[s]/empty[s] smem ring (TMA <-> consumers), rfull/rempty residual slabs (TMA <-> epilogue).
// N: accumulator columns (BN, or 2 BN in wide mode), the width of the wgmma instructions.  MMA: TM_MMA_* (the products
// issued per K slice), a template parameter so that no run-time branch sits between the wgmmas of a k-block.
template <int N, int MMA>
__global__ void __launch_bounds__(TM_THREADS, 1)
igemm_tma_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
                 const __grid_constant__ CUtensorMap tm_y, const __grid_constant__ CUtensorMap tm_r, const TmaGeom g) {
  extern __shared__ __align__(1024) uint8_t smem_dyn[];
  const uint32_t raw = smem_u32(smem_dyn);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* sm = smem_dyn + (base - raw);
  const TmaSmem L = tma_smem_layout(g.BN, g.stages, g.has_res != 0, g.direct != 0, g.x3 != 0, g.res_up2 != 0, g.res_inplace != 0,
                                    g.opairs);
  const uint32_t bar_full = base, bar_empty = base + 8 * TM_MAX_STAGES;
  const uint32_t bar_rfull = bar_empty + 8 * TM_MAX_STAGES, bar_rempty = bar_rfull + 16;     // two residual buffers

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int cchunks = g.Cin / 64;
  const int num_kb = g.KHW * cchunks;
  // images are the slowest tile coordinate, so the tiles of images < n are a prefix of the tile sequence
  const int tiles_n = g.n_dev ? (min(max(*g.n_dev, 0), g.N) + g.bn - 1) / g.bn : g.tiles_n;
  const long long m_tiles = (long long)g.tiles_w * g.tiles_h * tiles_n;
  const long long num_tiles = m_tiles * g.n_tiles;
  const uint32_t box_bytes = (uint32_t)(g.bw * g.bh * g.bn) * 128u;

  if (tid == 0) {
    for (int s = 0; s < g.stages; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, TM_EPI_WARPS);
    }
    for (int b = 0; b < 2; ++b) {
      mbar_init(bar_rfull + 8 * b, 1);
      mbar_init(bar_rempty + 8 * b, g.res_inplace ? 1 : TM_EPI_WARPS);
    }
    fence_mbar_init();
  } else if (warp == TM_WARP_TMA && lane == 0) {
    prefetch_tmap(&tm_x);
    prefetch_tmap(&tm_w);
    prefetch_tmap(&tm_y);
    if (g.has_res || (g.stem && g.x3)) prefetch_tmap(&tm_r);
  }
  __syncthreads();

  if (warp == TM_WARP_TMA) {
    // =============================== OPERAND LOADS ===============================
    if (lane == 0) {
      // ring position / phase are running counters: no division on the per-k-block path of this single thread
      uint32_t s = 0, ph = 0;
      uint32_t a_dst = base + L.stages;
      const uint32_t tx_bytes = (g.x3 ? 2u * box_bytes : box_bytes) + L.b_bytes;
      for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int nt = (int)(tile % g.n_tiles);
        const long long mt = tile / g.n_tiles;
        const int w0 = (int)(mt % g.tiles_w) * g.bw;
        const int h0 = (int)((mt / g.tiles_w) % g.tiles_h) * g.bh;
        const int i0 = (int)(mt / ((long long)g.tiles_w * g.tiles_h)) * g.bn;
        const int n0 = nt * g.BN;
        int kbr = 0, cc = 0, kj = 0;
        int cw = w0 - g.pw, ch = h0 - g.ph;         // box origin of the current tap
        for (int kb = 0; kb < num_kb; ++kb) {
          const uint32_t bf = bar_full + 8 * s;
          mbar_wait(bar_empty + 8 * s, ph ^ 1u);
          mbar_arrive_expect_tx(bf, tx_bytes);
          if (g.stem)   // k-block = filter row ky: 8 pixels x 8 channels per output pixel, input row 2*ho + ky of the padded image
            tma_load_5d(a_dst, &tm_x, bf, 0, w0, kbr & 1, h0 + (kbr >> 1), i0);
          else
            tma_load_4d(a_dst, &tm_x, bf, cc * 64, cw, ch, i0);
          tma_load_2d(a_dst + L.a_bytes, &tm_w, bf, kbr * 64, n0);
          if (g.x3) {
            if (g.stem)   // pair stem: the lo plane of the packed image has its own tensor map (tm_r is free: no residual)
              tma_load_5d(a_dst + L.a_half, &tm_r, bf, 0, w0, kbr & 1, h0 + (kbr >> 1), i0);
            else
              tma_load_4d(a_dst + L.a_half, &tm_x, bf, g.x_lo + cc * 64, cw, ch, i0);
            tma_load_2d(a_dst + L.a_bytes + L.b_half, &tm_w, bf, kbr * 64, g.w_lo + n0);
          }
          ++kbr;
          if (++cc == cchunks) {
            cc = 0; cw += g.dw;
            if (++kj == g.kw) { kj = 0; cw = w0 - g.pw; ch += g.dh; }
          }
          a_dst += L.stage_bytes;
          if (++s == (uint32_t)g.stages) { s = 0; ph ^= 1u; a_dst = base + L.stages; }
        }
      }
    }
    __syncwarp();
  } else if (warp == TM_WARP_RES) {
    // =============================== RESIDUAL LOADS ===============================
    if (lane == 0 && g.has_res) {
      uint32_t ti_local = 0;
      const int slabs = g.BN / 64;
      for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++ti_local) {
        const int nt = (int)(tile % g.n_tiles);
        const long long mt = tile / g.n_tiles;
        const int w0 = (int)(mt % g.tiles_w) * g.bw;
        const int h0 = (int)((mt / g.tiles_w) % g.tiles_h) * g.bh;
        const int i0 = (int)(mt / ((long long)g.tiles_w * g.tiles_h)) * g.bn;
        // residual slabs are double-buffered: tile t+1's residual streams in from HBM while tile t's epilogue runs
        const uint32_t rb = ti_local & 1u, ruse = ti_local >> 1;
        const uint32_t rdst = base + L.res + rb * (uint32_t)slabs * TM_SLAB_BYTES;
        mbar_wait(bar_rempty + 8 * rb, (ruse & 1u) ^ 1u);
        if (g.x3) {
          // pair mode: (hi, lo) slab per 64 channels; in-place mode lands them in this tile's output slab pairs
          const uint32_t lo_off = g.res_inplace ? (uint32_t)TM_SLAB_BYTES : L.res_slab;
          const uint32_t pdst = g.res_inplace ? base + L.out + rb * (uint32_t)slabs * 2u * TM_SLAB_BYTES
                                              : base + L.res + rb * (uint32_t)slabs * 2u * L.res_slab;
          mbar_arrive_expect_tx(bar_rfull + 8 * rb, (g.res_up2 ? box_bytes / 4 : box_bytes) * (uint32_t)slabs * 2u);
          for (int s = 0; s < slabs; ++s) {
            const int c = pair_chan(nt * g.BN + s * 64, g.pg);
            tma_load_4d(pdst + (uint32_t)s * 2u * lo_off, &tm_r, bar_rfull + 8 * rb, c, w0 >> g.res_up2, h0 >> g.res_up2, i0);
            tma_load_4d(pdst + (uint32_t)s * 2u * lo_off + lo_off, &tm_r, bar_rfull + 8 * rb, c + g.pg, w0 >> g.res_up2,
                        h0 >> g.res_up2, i0);
          }
          continue;
        }
        // res_up2: the box of the half-resolution map that covers this tile is (bw/2, bh/2) at (w0/2, h0/2)
        mbar_arrive_expect_tx(bar_rfull + 8 * rb, (g.res_up2 ? box_bytes / 4 : box_bytes) * (uint32_t)slabs);
        for (int s = 0; s < slabs; ++s)
          tma_load_4d(rdst + s * TM_SLAB_BYTES, &tm_r, bar_rfull + 8 * rb, nt * g.BN + s * 64, w0 >> g.res_up2,
                      h0 >> g.res_up2, i0);
      }
    }
    __syncwarp();
  } else {
    // =============================== CONSUMERS (warps 0-7) ===============================
    const int wg = warp >> 2;
    const uint32_t dhi = wg_desc_hi(1024);
    const uint32_t a_row0 = (uint32_t)wg * 64u * 128u;       // this warpgroup's 64 rows of the A tile
    const uint32_t ah16 = L.a_half >> 4;       // pair mode: lo A tile offset (descriptor units)
    float* accbuf = reinterpret_cast<float*>(sm + L.acc);
    constexpr int SW = MMA == TM_MMA_WIDE ? N / 2 : N;        // staged columns (= BN)
    // the pair slab epilogue reads the fragments; the bf16-stream and direct-store epilogues read staged rows
    const bool staged = MMA != TM_MMA_WIDE || g.direct;
    float d[N / 2];
    uint32_t s = 0, ph = 0;
    // main loop of one tile, then (staged epilogues) its accumulators -> staging rows (all eight warps take part)
    auto mainloop = [&]() {
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(bar_full + 8 * s, ph);
        const uint32_t st0 = base + L.stages + s * L.stage_bytes;
        const uint32_t a = wg_desc_lo(st0 + a_row0), b = wg_desc_lo(st0 + L.a_bytes);
        wgmma_fence();
#pragma unroll
        for (uint32_t k = 0; k < 4; ++k) {       // 16 bf16 = 32 bytes = 2 descriptor units inside the swizzle span
          const uint32_t acc = (kb | k) ? 1u : 0u;
          if constexpr (MMA == TM_MMA_WIDE) {   // hi * [hi ; lo] -> columns [0, 2 BN), lo * hi -> columns [0, BN)
            Wgmma<N>::mma(d, wg_desc(a + 2 * k, dhi), wg_desc(b + 2 * k, dhi), acc);
            Wgmma<N / 2>::mma(*reinterpret_cast<float(*)[N / 4]>(&d[0]), wg_desc(a + ah16 + 2 * k, dhi), wg_desc(b + 2 * k, dhi), 1u);
          } else {
            Wgmma<N>::mma(d, wg_desc(a + 2 * k, dhi), wg_desc(b + 2 * k, dhi), acc);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();                         // the previous k-block's wgmmas have read their stage
        wgmma_fence_acc(d);
        if (prev >= 0 && lane == 0) mbar_arrive(bar_empty + 8 * prev);
        prev = (int)s;
        if (++s == (uint32_t)g.stages) { s = 0; ph ^= 1u; }
      }
      wgmma_wait<0>();
      wgmma_fence_acc(d);
      if (prev >= 0 && lane == 0) mbar_arrive(bar_empty + 8 * prev);
      if constexpr (MMA == TM_MMA_WIDE) {        // hi*hi + lo*hi (columns [0, BN)) + hi*lo (columns [BN, 2 BN)): same thread
        // Zeroing the folded group ends its live range here (the next tile's first wgmma overwrites it, but the compiler
        // cannot see that): with N = 256 the epilogue then holds 64 accumulators instead of 128 and nothing spills.
#pragma unroll
        for (int i = 0; i < N / 4; ++i) { d[i] += d[N / 4 + i]; d[N / 4 + i] = 0.f; }
      }
      if (staged) {
        named_bar(3, 256);                  // the previous tile's epilogue has read the staging rows
        acc_stage_sw<N, SW>(d, accbuf, wg * 64);
        named_bar(3, 256);
      }
    };
    const int q = warp & 3, half = warp >> 2;
    const int row = q * 32 + lane;
    const uint32_t trow = smem_u32(accbuf + (size_t)row * SW);
    const int units = g.BN / 32;                       // 32-column units of the accumulator
    const int upw = units >= 4 ? units / 2 : 1;        // units per half (BN = 64: one each)
    const int bar_id = g.BN == 64 ? 1 : 1 + half;
    const int bar_cnt = g.BN == 64 ? 256 : 128;
    const bool leader = (g.BN == 64 ? warp == 0 : q == 0) && lane == 0;
    const uint32_t out_slab = base + L.out + (g.BN == 64 ? 0u : (uint32_t)half * TM_SLAB_BYTES);
    const uint32_t sw_row = (uint32_t)row * 128u;
    const uint32_t rx = (uint32_t)(row & 7);
    auto res_row = [&](int r) {                        // row of the residual slab that accumulator row r reads
      if (!g.res_up2) return r;
      const int w = r % g.bw, h = (r / g.bw) % g.bh, n = r / (g.bw * g.bh);
      return (w >> 1) + (g.bw >> 1) * ((h >> 1) + (g.bh >> 1) * n);
    };
    const int rrow = res_row(row);
    const uint32_t rs_row = (uint32_t)rrow * 128u, rrx = (uint32_t)(rrow & 7);
    // pair slab epilogue: byte offsets of this thread's two fragment rows in a slab, and of the residual rows they read
    uint32_t fr_row[2], fr_res[2], fr_rx[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = wg * 64 + 16 * (warp & 3) + (lane >> 2) + 8 * h, rr = res_row(r);
      fr_row[h] = (uint32_t)r * 128u; fr_res[h] = (uint32_t)rr * 128u; fr_rx[h] = (uint32_t)(rr & 7);
    }
    uint32_t ti_local = 0, oc = 0;
    for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++ti_local) {
      const int nt = (int)(tile % g.n_tiles);
      const long long mt = tile / g.n_tiles;
      const int w0 = (int)(mt % g.tiles_w) * g.bw;
      const int h0 = (int)((mt / g.tiles_w) % g.tiles_h) * g.bh;
      const int i0 = (int)(mt / ((long long)g.tiles_w * g.tiles_h)) * g.bn;
      const int n0 = nt * g.BN;
      const uint32_t buf = ti_local & 1u, use = ti_local >> 1;
      mainloop();
      if (g.has_res) mbar_wait(bar_rfull + 8 * buf, use & 1u);
      if (g.direct) {
        // thread = accumulator row = one output pixel of the box; the two halves split the columns
        const int wq = row % g.bw, hq = (row / g.bw) % g.bh, nq = row / (g.bw * g.bh);
        const int wo = w0 + wq, ho = h0 + hq, ni = i0 + nq;
        const bool ok = nq < g.bn && wo < g.Wo && ho < g.Ho && ni < g.N;
        const size_t HoWo = (size_t)g.Ho * g.Wo;
        const size_t pix = ((size_t)ni * g.Ho + ho) * g.Wo + wo;
        const int cbeg = half * (g.BN / 2), cend = cbeg + g.BN / 2;
        for (int cb = cbeg; cb < cend; cb += 16) {
          uint32_t v[16];
          acc_ld16_sw(trow, row, cb, v);
          const int co0 = n0 + cb;
          if (!ok || co0 >= g.Cout) continue;
#pragma unroll
          for (int e = 0; e < 16; ++e) {
            const int co = co0 + e;
            if (co >= g.Cout) break;
            float o = __uint_as_float(v[e]);
            if (g.bias) o += __ldg(g.bias + co);
            if (g.relu) o = fmaxf(o, 0.f);
            if (g.sig_from >= 0 && co >= g.sig_from) o = 1.f / (1.f + expf(-o));
            const size_t oi = g.out_nhwc ? pix * g.Cout + co : ((size_t)ni * g.Cout + co) * HoWo + (size_t)ho * g.Wo + wo;
            if (g.y_bf16) reinterpret_cast<__nv_bfloat16*>(g.y)[oi] = __float2bfloat16_rn(o);
            else reinterpret_cast<float*>(g.y)[oi] = o;
          }
        }
        continue;
      }
      if constexpr (MMA == TM_MMA_WIDE) {
        // ---- pair slab epilogue, on the fragments: all eight warps share one 64-channel (hi, lo) slab pair at a time, each
        //      thread holds rows fr[h] and, per 8-column group j of the slab, columns 8 j + cq + {0, 1}.
        //      fp32 result -> hi = bf16(o), lo = bf16(o - hi) -> one bf16x2 word per slab, at chunk j ^ (row & 7): the 8 rows
        //      of a store instruction hit 8 distinct chunks (conflict-free) -> two TMA stores per slab pair ----
        const bool lead = warp == 0 && lane == 0;
        const uint32_t cq4 = (uint32_t)(lane & 3) * 4u;      // byte offset of the column pair inside a 16-byte chunk
        const uint32_t fx = (uint32_t)(lane >> 2);           // fragment row & 7 (both rows)
#pragma unroll
        for (int sl = 0; sl < SW / 64; ++sl, ++oc) {
          uint32_t ob;
          if (g.res_inplace) {
            ob = base + L.out + (buf * (uint32_t)(SW / 64) + (uint32_t)sl) * 2u * TM_SLAB_BYTES;   // holds this slab's residual
          } else {
            ob = base + L.out + (g.opairs == 2 ? (oc & 1u) : 0u) * 2u * TM_SLAB_BYTES;
            if (lead) {                             // the stores that last used this pair have finished reading it
              if (g.opairs == 2) bulk_wait_read1(); else bulk_wait_read0();
            }
            named_bar(1, 256);
          }
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int i = 8 * sl + j;                        // fragment column group
            float2 bv = make_float2(0.f, 0.f);
            if (g.bias) bv = __ldg(reinterpret_cast<const float2*>(g.bias + n0 + 8 * i) + (lane & 3));
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float a = d[4 * i + 2 * h], b = d[4 * i + 2 * h + 1];
              const uint32_t oa = ob + fr_row[h] + (((uint32_t)j ^ fx) << 4) + cq4;
              if (g.bias) { a += bv.x; b += bv.y; }
              if (g.has_res) {
                uint32_t hw, lw;
                if (g.res_inplace) { hw = lds32(oa); lw = lds32(oa + TM_SLAB_BYTES); }
                else {
                  const uint32_t ra = base + L.res + (buf * (uint32_t)(SW / 64) + (uint32_t)sl) * 2u * L.res_slab + fr_res[h];
                  hw = lds32(ra + (((uint32_t)j ^ fr_rx[h]) << 4) + cq4);
                  lw = lds32(ra + L.res_slab + (((uint32_t)j ^ fr_rx[h]) << 4) + cq4);
                }
                a += pair_x(hw, lw);
                b += pair_y(hw, lw);
              }
              if (g.relu) { a = fmaxf(a, 0.f); b = fmaxf(b, 0.f); }
              uint32_t hw, lw;
              split_pair2(a, b, hw, lw);
              sts32(oa, hw);
              sts32(oa + TM_SLAB_BYTES, lw);
            }
          }
          fence_proxy_async();
          named_bar(1, 256);
          if (lead) {
            const int c = pair_chan(n0 + sl * 64, g.pg);
            tma_store_4d(&tm_y, ob, c, w0, h0, i0);
            tma_store_4d(&tm_y, ob + TM_SLAB_BYTES, c + g.pg, w0, h0, i0);
            bulk_commit();
          }
        }
        __syncwarp();
        if (lane == 0 && g.has_res && !g.res_inplace) mbar_arrive(bar_rempty + 8 * buf);
        if (g.res_inplace && lead) {     // the slab pairs of this tile may be refilled once their stores have been read out
          bulk_wait_read0();
          mbar_arrive(bar_rempty + 8 * buf);
        }
      } else {
        for (int ui = 0; ui < upw; ++ui) {
          const int u = half * upw + ui;
          const int slab = u >> 1;
          const uint32_t jb = (uint32_t)(u & 1) * 4u;     // first 16-byte chunk of this unit inside the slab row
          uint32_t v0[16], v1[16];
          acc_ld16_sw(trow, row, u * 32, v0);
          acc_ld16_sw(trow, row, u * 32 + 16, v1);
          if ((u & 1) == 0 || g.BN == 64) {
            // the output slab is about to be overwritten: its previous TMA store must have finished reading it
            if (leader) bulk_wait_read0();
            named_bar(bar_id, bar_cnt);
          }
          float o[32];
  #pragma unroll
          for (int e = 0; e < 16; ++e) { o[e] = __uint_as_float(v0[e]); o[16 + e] = __uint_as_float(v1[e]); }
          if (g.bias) {
            const float4* bp = reinterpret_cast<const float4*>(g.bias + n0 + u * 32);
  #pragma unroll
            for (int e = 0; e < 8; ++e) {
              const float4 b4 = __ldg(bp + e);
              o[4 * e] += b4.x; o[4 * e + 1] += b4.y; o[4 * e + 2] += b4.z; o[4 * e + 3] += b4.w;
            }
          }
          if (g.has_res) {
            const uint32_t rs = base + L.res + (buf * (uint32_t)(g.BN / 64) + (uint32_t)slab) * TM_SLAB_BYTES + rs_row;
  #pragma unroll
            for (int c = 0; c < 4; ++c) {
              const uint4 rv = lds128(rs + (((jb + c) ^ rrx) << 4));
              const uint32_t rw[4] = {rv.x, rv.y, rv.z, rv.w};
  #pragma unroll
              for (int e = 0; e < 4; ++e) {
                o[c * 8 + 2 * e] += bf16x2_x(rw[e]);
                o[c * 8 + 2 * e + 1] += bf16x2_y(rw[e]);
              }
            }
          }
          if (g.relu) {
  #pragma unroll
            for (int e = 0; e < 32; ++e) o[e] = fmaxf(o[e], 0.f);
          }
  #pragma unroll
          for (int c = 0; c < 4; ++c) sts128(out_slab + sw_row + (((jb + c) ^ rx) << 4), pack_bf16x8(o + c * 8));
          if ((u & 1) == 1 || g.BN == 64) {
            fence_proxy_async();                 // generic-proxy smem writes -> visible to the TMA store
            named_bar(bar_id, bar_cnt);
            if (leader) {
              tma_store_4d(&tm_y, out_slab, n0 + slab * 64, w0, h0, i0);
              bulk_commit();
            }
          }
        }
        __syncwarp();
        if (lane == 0 && g.has_res) mbar_arrive(bar_rempty + 8 * buf);
      }
    }
    if (leader || (g.x3 && warp == 0 && lane == 0)) bulk_wait0();
  }
}

// ----------------------------------------------------------------------------------------------
// host side: tensor maps, tile geometry, launch
// ----------------------------------------------------------------------------------------------
// bf16 tensor, innermost dimension first; box[0] = 64 elements = one 128-byte swizzle span
static bool encode_bf16(EncodeTiledFn enc, CUtensorMap* tm, const void* ptr, int rank, const cuuint64_t* dims,
                        const cuuint32_t* box, const cuuint64_t* byte_strides = nullptr) {
  cuuint64_t strides[5];
  cuuint64_t acc = 2;
  for (int i = 0; i + 1 < rank; ++i) { acc *= dims[i]; strides[i] = byte_strides ? byte_strides[i] : acc; }
  const cuuint32_t es[5] = {1, 1, 1, 1, 1};
  return enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides, box, es,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Output-pixel box (bw, bh, bn) with bw*bh*bn <= 128: fewest tiles, then smallest input halo, then widest rows.
static void tma_pick_box(int N, int Ho, int Wo, int kh, int kw, int dh, int dw, bool even, int* bw_o, int* bh_o, int* bn_o) {
  long long best_tiles = -1, best_halo = 0;
  int bbw = 1, bbh = 1, bbn = 1;
  const int wmax = Wo < 128 ? Wo : 128;
  for (int bw = 1; bw <= wmax; ++bw) {
    if (Wo > 32 && (bw & (bw - 1))) continue;     // large maps: power-of-two widths only (keeps the search tiny)
    if (even && (bw & 1)) continue;
    const int hmax = (128 / bw) < Ho ? (128 / bw) : Ho;
    for (int bh = 1; bh <= hmax; ++bh) {
      if (even && (bh & 1)) continue;
      int bn = 128 / (bw * bh);
      if (bn > N) bn = N;
      if (bn < 1) continue;
      const long long tiles = (long long)((Wo + bw - 1) / bw) * ((Ho + bh - 1) / bh) * ((N + bn - 1) / bn);
      const long long halo = (long long)(bw + (kw - 1) * dw) * (bh + (kh - 1) * dh) * bn;
      if (best_tiles < 0 || tiles < best_tiles || (tiles == best_tiles && (halo < best_halo || (halo == best_halo && bw > bbw)))) {
        best_tiles = tiles; best_halo = halo; bbw = bw; bbh = bh; bbn = bn;
      }
    }
  }
  *bw_o = bbw; *bh_o = bbh; *bn_o = bbn;
}

template <int N, int MMA>
static int tma_launch_n(dim3 grid, size_t smem, cudaStream_t stream, const CUtensorMap& tm_x, const CUtensorMap& tm_w,
                        const CUtensorMap& tm_y, const CUtensorMap& tm_r, const TmaGeom& g) {
  static ups::PerDeviceOnce configured;     // opt in to 227 KB once per device (outside CUDA-graph capture)
  if (configured.need())
    UPS_CUDA(cudaFuncSetAttribute(igemm_tma_kernel<N, MMA>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  igemm_tma_kernel<N, MMA><<<grid, TM_THREADS, smem, stream>>>(tm_x, tm_w, tm_y, tm_r, g);
  UPS_CHECK_LAUNCH();
  return 0;
}
// kernel instance for the N tile BN and the geometry's products: bf16 stream N = BN; pairs (wide) N = 2 BN
static int tma_launch(int BN, dim3 grid, size_t smem, cudaStream_t stream, const CUtensorMap& tm_x, const CUtensorMap& tm_w,
                      const CUtensorMap& tm_y, const CUtensorMap& tm_r, const TmaGeom& g) {
  if (g.wide) {
    if (BN == 32) return tma_launch_n<64, TM_MMA_WIDE>(grid, smem, stream, tm_x, tm_w, tm_y, tm_r, g);
    if (BN == 64) return tma_launch_n<128, TM_MMA_WIDE>(grid, smem, stream, tm_x, tm_w, tm_y, tm_r, g);
    if (BN == 128) return tma_launch_n<256, TM_MMA_WIDE>(grid, smem, stream, tm_x, tm_w, tm_y, tm_r, g);
  } else {
    if (BN == 32) return tma_launch_n<32, TM_MMA_BF16>(grid, smem, stream, tm_x, tm_w, tm_y, tm_r, g);
    if (BN == 64) return tma_launch_n<64, TM_MMA_BF16>(grid, smem, stream, tm_x, tm_w, tm_y, tm_r, g);
    if (BN == 128) return tma_launch_n<128, TM_MMA_BF16>(grid, smem, stream, tm_x, tm_w, tm_y, tm_r, g);
  }
  return UPSNET_E_UNSUPPORTED;
}

// Ring depth and output slab pairs for an N tile: the deepest ring that fits (<= TM_MAX_STAGES, >= 2); pair mode: when two
// alternating output slab pairs leave fewer than four stages (or do not fit at all), one pair buys stages -- the main loop
// needs the depth more than the epilogue does.
static bool tma_fit(int BN, bool has_res, bool direct, bool pair, bool res_up2, bool res_inplace, int* stages, int* opairs,
                    TmaSmem* L) {
  const uint32_t cap = 227 * 1024 - 1024;
  auto lay = [&](int st, int op) { return tma_smem_layout(BN, st, has_res, direct, pair, res_up2, res_inplace, op); };
  int st = TM_MAX_STAGES, op = 2;
  while (st > 2 && lay(st, op).total > cap) --st;
  if (pair && !direct && !res_inplace && (st < 4 || lay(st, op).total > cap)) {
    int st1 = 4;
    while (st1 > 2 && lay(st1, 1).total > cap) --st1;
    if (st1 > st || lay(st, op).total > cap) { st = st1; op = 1; }
  }
  *stages = st; *opairs = op; *L = lay(st, op);
  return L->total <= cap;
}

// N tile of the next launches: 0 = chosen per launch (below), 64 or 128 = that N tile wherever Cout rounded up allows it and
// it fits (else the launch narrows it as it does its own choice).  For tests and tuning: lets one process compare the tiles.
static int g_tma_force_bn = 0;

int launch_igemm_tma(const TcParams& p, const void* packed, cudaStream_t stream) {
  if (p.no_tma || p.offset) return UPSNET_E_UNSUPPORTED;
  // precision bf16 runs on bf16 activations, precision bf16x3 on hi/lo bf16 pairs (same tile pipeline, three MMAs)
  const bool pair = p.x_pair != 0;
  if (pair != (p.x3 != 0) || (!pair && !p.x_bf16)) return UPSNET_E_UNSUPPORTED;
  if (p.y_pair && (!pair || !p.out_nhwc || (p.Cout % 64) != 0)) return UPSNET_E_UNSUPPORTED;
  if (pair && p.y_bf16) return UPSNET_E_UNSUPPORTED;     // pair in -> pair (slab epilogue) or fp32 (direct epilogue) out
  const int pg = p.y_pair ? (p.pair_group > 0 ? p.pair_group : p.Cout) : 0;
  if (p.y_pair && ((pg % 64) != 0 || (p.Cout % pg) != 0)) return UPSNET_E_UNSUPPORTED;
  // slab epilogue (TMA store): bf16 / pair NHWC output with Cout % 64 == 0; everything else without a residual goes
  // through the direct-store epilogue (small heads: Cout 9..45, fp32 planes)
  const bool direct = (!p.y_bf16 && !p.y_pair) || !p.out_nhwc || (p.Cout % 64) != 0;
  if (p.sig_from >= 0 && !direct) return UPSNET_E_UNSUPPORTED;
  if (direct && (p.residual || p.Cout > 256)) return UPSNET_E_UNSUPPORTED;
  if (p.res_up2 && (!p.residual || (p.Ho & 1) || (p.Wo & 1))) return UPSNET_E_UNSUPPORTED;
  // stride > 1 only for 1x1 / pad 0 (the ResNet down-sampling convs): the input is then addressed through a
  // strided VIEW (every sh-th row, sw-th pixel) and the layer is a stride-1 1x1 convolution of that view
  const bool strided = p.sh != 1 || p.sw != 1;
  if (strided && (p.kh != 1 || p.kw != 1 || p.ph != 0 || p.pw != 0)) return UPSNET_E_UNSUPPORTED;
  if ((p.Cin % 64) || (!direct && (p.Cout % 64)) || p.kh * p.kw > 49) return UPSNET_E_UNSUPPORTED;
  if ((((uintptr_t)p.x) & 15) || (((uintptr_t)p.y) & 15) || (((uintptr_t)packed) & 15) || (p.residual && (((uintptr_t)p.residual) & 15)))
    return UPSNET_E_UNSUPPORTED;
  if (p.bias && (((uintptr_t)p.bias) & 15)) return UPSNET_E_UNSUPPORTED;
  EncodeTiledFn enc = tma_encoder();
  if (!enc) return UPSNET_E_UNSUPPORTED;
  const int sms = num_sms();
  TmaGeom g{};
  g.bias = p.bias;
  g.N = p.N; g.Ho = p.Ho; g.Wo = p.Wo; g.Cout = p.Cout; g.Cin = p.Cin;
  g.kw = p.kw; g.KHW = p.kh * p.kw; g.ph = p.ph; g.pw = p.pw; g.dh = p.dh; g.dw = p.dw;
  g.relu = p.relu; g.has_res = p.residual ? 1 : 0; g.res_up2 = p.res_up2 ? 1 : 0; g.sig_from = p.sig_from;
  g.n_dev = p.n_dev;
  tma_pick_box(p.N, p.Ho, p.Wo, p.kh, p.kw, p.dh, p.dw, g.res_up2 != 0, &g.bw, &g.bh, &g.bn);
  g.tiles_w = (p.Wo + g.bw - 1) / g.bw;
  g.tiles_h = (p.Ho + g.bh - 1) / g.bh;
  g.tiles_n = (p.N + g.bn - 1) / g.bn;
  const long long m_tiles = (long long)g.tiles_w * g.tiles_h * g.tiles_n;
  const int Cout_pad = cout_pad(p.Cout);
  // N tile <= 128: the accumulators are m64nBN register fragments of two warpgroups (bf16 stream: 64 floats per thread at
  // 128; pairs: m64n2BN, 128 floats per thread at 128)
  int BN = (Cout_pad % 128 == 0) ? 128 : (Cout_pad % 64 == 0 ? 64 : 32);
  g.x3 = pair ? 1 : 0; g.x_lo = p.Cin; g.w_lo = Cout_pad; g.pg = pg;
  g.res_inplace = (pair && g.has_res && !g.res_up2) ? 1 : 0;
  g.opairs = 2;
  if (g_tma_force_bn && Cout_pad % g_tma_force_bn == 0) {
    BN = g_tma_force_bn;
  } else {
    // N tile: as wide as possible (operand bytes per flop fall with BN) while ~2/3 of the SMs still get a tile
    while (BN > 64 && m_tiles * (Cout_pad / BN) < 88) BN /= 2;
  }
  g.direct = direct ? 1 : 0; g.y_bf16 = p.y_bf16; g.out_nhwc = p.out_nhwc; g.y = p.y;
  TmaSmem L;
  bool ok = tma_fit(BN, g.has_res != 0, direct, pair, g.res_up2 != 0, g.res_inplace != 0, &g.stages, &g.opairs, &L);
  // a narrower N tile frees operand, slab and staging space.  Pairs: a 2-stage ring at N = 128 loses to a deeper one at 64
  // (measured on H100 SXM, bf16x3 bench: N = 128 pair tiles with 2 stages ran the dense conv family 8 % slower than N = 64)
  while (BN > 64 && (!ok || (pair && g.stages < 3))) {
    BN /= 2;
    ok = tma_fit(BN, g.has_res != 0, direct, pair, g.res_up2 != 0, g.res_inplace != 0, &g.stages, &g.opairs, &L);
  }
  if (!ok) return UPSNET_E_UNSUPPORTED;
  g.BN = BN;
  g.n_tiles = Cout_pad / BN;

  const int Kp = g.KHW * p.Cin;
  CUtensorMap tm_x, tm_w, tm_y, tm_r;
  {
    const cuuint64_t xm = pair ? 2 : 1;      // pair tensors carry 2*C channels per pixel (hi plane, lo plane)
    const cuuint64_t dx[4] = {(cuuint64_t)p.Cin * xm, (cuuint64_t)(strided ? p.Wo : p.W), (cuuint64_t)(strided ? p.Ho : p.H),
                              (cuuint64_t)p.N};
    const cuuint64_t sx[3] = {(cuuint64_t)p.sw * p.Cin * 2 * xm, (cuuint64_t)p.sh * p.W * p.Cin * 2 * xm,
                              (cuuint64_t)p.H * p.W * p.Cin * 2 * xm};
    const cuuint64_t dy[4] = {(cuuint64_t)p.Cout * xm, (cuuint64_t)p.Wo, (cuuint64_t)p.Ho, (cuuint64_t)p.N};
    const cuuint64_t dwt[2] = {(cuuint64_t)Kp, (cuuint64_t)Cout_pad * xm};       // the packed weights ARE [hi plane][lo plane]
    const cuuint32_t box[4] = {64, (cuuint32_t)g.bw, (cuuint32_t)g.bh, (cuuint32_t)g.bn};
    const cuuint32_t boxw[2] = {64, (cuuint32_t)BN};
    if (!encode_bf16(enc, &tm_x, p.x, 4, dx, box, sx)) return UPSNET_E_UNSUPPORTED;
    if (!encode_bf16(enc, &tm_w, packed, 2, dwt, boxw)) return UPSNET_E_UNSUPPORTED;
    if (direct) {   // no TMA store / residual in the direct-store epilogue: the two maps are placeholders
      tm_y = tm_x;
      tm_r = tm_x;
    } else {
    if (!encode_bf16(enc, &tm_y, p.y, 4, dy, box)) return UPSNET_E_UNSUPPORTED;
    if (g.res_up2) {
      const cuuint64_t dr[4] = {(cuuint64_t)p.Cout * xm, (cuuint64_t)(p.Wo / 2), (cuuint64_t)(p.Ho / 2), (cuuint64_t)p.N};
      const cuuint32_t boxr[4] = {64, (cuuint32_t)(g.bw / 2), (cuuint32_t)(g.bh / 2), (cuuint32_t)g.bn};
      if (!encode_bf16(enc, &tm_r, p.residual, 4, dr, boxr)) return UPSNET_E_UNSUPPORTED;
    } else if (!encode_bf16(enc, &tm_r, p.residual ? p.residual : p.y, 4, dy, box)) {
      return UPSNET_E_UNSUPPORTED;
    }
    }
  }
  const long long num_tiles = m_tiles * g.n_tiles;
  if (num_tiles <= 0) return 0;
  g.wide = pair ? 1 : 0;    // pair stream: two wgmma per K slice (see TmaGeom::wide)
  dim3 grid((unsigned)(num_tiles < sms ? num_tiles : sms));
  return tma_launch(BN, grid, L.total + 1024, stream, tm_x, tm_w, tm_y, tm_r, g);
}


// ----------------------------------------------------------------------------------------------
// RGB stem (models/resnet.py:155-162 conv1: 7x7 / stride 2 / pad 3, Cin = 3) on the TMA kernel.
// The fp32 NCHW image is first packed to a zero-padded bf16 NHWC8 image (stem_pack_image_kernel); the eight input
// pixels x 8 channels an output pixel needs from filter row ky are then 128 contiguous bytes, consecutive output
// pixels start 32 bytes apart, and even / odd input rows are split by a parity dimension -- a 5-D tensor map
// (64 el, Wo @32 B, 2 @pitch, Hp/2 @2*pitch, N) whose boxes ARE the im2col tiles, one k-block per filter row.
// Weights are packed [Cout][ky][8 px][8 ch] with zeros for kx >= kw and c >= Cin (K = 64*kh).
// ----------------------------------------------------------------------------------------------
__global__ void stem_pack_image_kernel(const float* __restrict__ x, uint4* __restrict__ xp, uint4* __restrict__ xp_lo, int N, int C,
                                       int H, int W, int pad, int Hp, int Wp) {
  const long long total = (long long)N * Hp * Wp;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(t % Wp);
    const long long rest = t / Wp;
    const int r = (int)(rest % Hp), n = (int)(rest / Hp);
    const int hi = r - pad, wi = c - pad;
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (hi >= 0 && hi < H && wi >= 0 && wi < W)
      for (int ch = 0; ch < C; ++ch) v[ch] = __ldg(x + (((size_t)n * C + ch) * H + hi) * W + wi);
    const uint4 o = pack_bf16x8(v);
    xp[t] = o;
    if (xp_lo) xp_lo[t] = pair_lo8(v, o);     // pair stem: second plane = bf16(v - hi)
  }
}

__global__ void stem_pack_weight_kernel(const float* __restrict__ w, int Cout, int Cin, int kh, int kw,
                                        __nv_bfloat16* __restrict__ packed) {
  const int total = Cout * kh * 64;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int c = i & 7, kx = (i >> 3) & 7, ky = (i >> 6) % kh, co = i / (64 * kh);
    const float v = (c < Cin && kx < kw) ? w[(((size_t)co * Cin + c) * kh + ky) * kw + kx] : 0.f;
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    packed[i] = h;
    packed[total + i] = l;      // lo plane (pair stem)
  }
}

static void stem_geometry(int H, int W, int kh, int kw, int pad, int* Ho, int* Wo, int* Hp, int* Wp) {
  *Ho = (H + 2 * pad - kh) / 2 + 1;
  *Wo = (W + 2 * pad - kw) / 2 + 1;
  *Hp = 2 * (*Ho + (kh >> 1));
  *Wp = 2 * *Wo + 8;
}

// the zero-padded bf16 NHWC8 image (16 bytes per pixel): the hi plane, then the lo plane, which only the pair stem has
inline size_t stem_layout(int N, int Hp, int Wp, bool pair, void* base, uint4** hi, uint4** lo) {
  WsCarve c(base);
  const size_t pixels = (size_t)N * Hp * Wp;
  *hi = c.take<uint4>(pixels);
  *lo = pair ? c.take<uint4>(pixels) : nullptr;
  return c.bytes();
}

}  // namespace ups

extern "C" int upsnet_tma_set_tile_n(int bn) {
  if (bn != 0 && bn != 64 && bn != 128) return UPSNET_E_BADARG;
  ups::g_tma_force_bn = bn;
  return 0;
}

extern "C" int upsnet_stem_workspace_bytes(int N, int H, int W, int kh, int kw, int pad, size_t* bytes) {
  if (!bytes || N <= 0 || H <= 0 || W <= 0 || kh <= 0 || kw <= 0 || kw > 8 || pad < 0) return UPSNET_E_BADARG;
  int Ho, Wo, Hp, Wp;
  ups::stem_geometry(H, W, kh, kw, pad, &Ho, &Wo, &Hp, &Wp);
  if (Ho <= 0 || Wo <= 0) return UPSNET_E_BADARG;
  uint4 *hi, *lo;
  *bytes = ups::stem_layout(N, Hp, Wp, true, nullptr, &hi, &lo);
  return 0;
}

extern "C" int upsnet_stem_packed_weight_bytes(int Cout, int kh, size_t* bytes) {
  if (!bytes || Cout <= 0 || kh <= 0) return UPSNET_E_BADARG;
  *bytes = (size_t)Cout * kh * 64 * 2 * 2;   // bf16 hi plane + lo plane
  return 0;
}

extern "C" int upsnet_stem_pack_weight(const float* weight, int Cout, int Cin, int kh, int kw, void* packed, void* stream) {
  if (!weight || !packed || Cout <= 0 || Cin <= 0 || Cin > 8 || kh <= 0 || kw <= 0 || kw > 8) return UPSNET_E_BADARG;
  const int total = Cout * kh * 64;
  ups::stem_pack_weight_kernel<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(weight, Cout, Cin, kh, kw,
                                                                                         (__nv_bfloat16*)packed);
  UPS_CHECK_LAUNCH();
  return 0;
}

extern "C" int upsnet_stem_forward(const float* x, const void* packed_w, const float* bias, void* y, int N, int Cin, int H,
                                   int W, int Cout, int kh, int kw, int pad, int epi_flags, void* workspace,
                                   size_t workspace_bytes, void* stream) {
  using namespace ups;
  if (!x || !packed_w || !y || !workspace) return UPSNET_E_BADARG;
  if (N <= 0 || Cin <= 0 || Cin > 8 || H <= 0 || W <= 0 || kh <= 0 || kw <= 0 || kw > 8 || pad < 0) return UPSNET_E_BADARG;
  if ((Cout % 64) || Cout > 256 || kh > 16) return UPSNET_E_UNSUPPORTED;
  if ((((uintptr_t)y) & 15) || (((uintptr_t)packed_w) & 15) || (((uintptr_t)workspace) & 15)) return UPSNET_E_BADARG;
  if (bias && (((uintptr_t)bias) & 15)) return UPSNET_E_UNSUPPORTED;
  int Ho, Wo, Hp, Wp;
  stem_geometry(H, W, kh, kw, pad, &Ho, &Wo, &Hp, &Wp);
  if (Ho <= 0 || Wo <= 0) return UPSNET_E_BADARG;
  const bool pair = (epi_flags & UPSNET_EPI_STEM_PAIR) != 0;
  uint4 *x_hi, *x_lo;
  if (workspace_bytes < stem_layout(N, Hp, Wp, pair, workspace, &x_hi, &x_lo)) return UPSNET_E_WORKSPACE;
  EncodeTiledFn enc = tma_encoder();
  if (!enc) return UPSNET_E_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  TmaGeom g{};
  g.bias = bias;
  g.N = N; g.Ho = Ho; g.Wo = Wo; g.Cout = Cout; g.Cin = 64;
  g.kw = 1; g.KHW = kh; g.ph = 0; g.pw = 0; g.dh = 1; g.dw = 1;
  g.relu = (epi_flags & UPSNET_EPI_RELU) ? 1 : 0;
  g.sig_from = -1;
  g.stem = 1; g.y = y; g.y_bf16 = 1; g.out_nhwc = 1;
  g.x3 = pair ? 1 : 0; g.w_lo = Cout; g.pg = Cout; g.opairs = 2; g.x_lo = 0;
  tma_pick_box(N, Ho, Wo, 1, 1, 1, 1, false, &g.bw, &g.bh, &g.bn);
  g.tiles_w = (Wo + g.bw - 1) / g.bw;
  g.tiles_h = (Ho + g.bh - 1) / g.bh;
  g.tiles_n = (N + g.bn - 1) / g.bn;
  g.BN = (Cout % 128 == 0 && !pair) ? 128 : 64;
  g.n_tiles = Cout / g.BN;
  g.wide = pair ? 1 : 0;     // pair stem: two wgmma per K slice over [W_hi ; W_lo] (see TmaGeom::wide)
  TmaSmem L;
  if (!tma_fit(g.BN, false, false, pair, false, false, &g.stages, &g.opairs, &L)) return UPSNET_E_UNSUPPORTED;
  CUtensorMap tm_x, tm_w, tm_y, tm_lo;
  {
    const cuuint64_t pitch = (cuuint64_t)Wp * 16;
    const cuuint64_t dx[5] = {64, (cuuint64_t)Wo, 2, (cuuint64_t)(Hp / 2), (cuuint64_t)N};
    const cuuint64_t sx[4] = {32, pitch, 2 * pitch, (cuuint64_t)Hp * pitch};
    const cuuint32_t bx[5] = {64, (cuuint32_t)g.bw, 1, (cuuint32_t)g.bh, (cuuint32_t)g.bn};
    const cuuint64_t dwt[2] = {(cuuint64_t)kh * 64, (cuuint64_t)Cout * 2};       // hi plane rows, then lo plane rows
    const cuuint32_t bw2[2] = {64, (cuuint32_t)g.BN};
    const cuuint64_t dy[4] = {(cuuint64_t)Cout * (pair ? 2 : 1), (cuuint64_t)Wo, (cuuint64_t)Ho, (cuuint64_t)N};
    const cuuint32_t by[4] = {64, (cuuint32_t)g.bw, (cuuint32_t)g.bh, (cuuint32_t)g.bn};
    if (!encode_bf16(enc, &tm_x, x_hi, 5, dx, bx, sx)) return UPSNET_E_UNSUPPORTED;
    tm_lo = tm_x;
    if (pair && !encode_bf16(enc, &tm_lo, x_lo, 5, dx, bx, sx)) return UPSNET_E_UNSUPPORTED;
    if (!encode_bf16(enc, &tm_w, packed_w, 2, dwt, bw2)) return UPSNET_E_UNSUPPORTED;
    if (!encode_bf16(enc, &tm_y, y, 4, dy, by)) return UPSNET_E_UNSUPPORTED;
  }
  {
    const long long total = (long long)N * Hp * Wp;
    long long blocks = (total + 255) / 256;
    if (blocks > kNumSMs * 32) blocks = kNumSMs * 32;
    stem_pack_image_kernel<<<(unsigned)blocks, 256, 0, st>>>(x, x_hi, x_lo, N, Cin, H, W, pad, Hp, Wp);
    UPS_CHECK_LAUNCH();
  }
  const int sms = num_sms();
  const long long num_tiles = (long long)g.tiles_w * g.tiles_h * g.tiles_n * g.n_tiles;
  dim3 grid((unsigned)(num_tiles < sms ? num_tiles : sms));
  return tma_launch(g.BN, grid, L.total + 1024, st, tm_x, tm_w, tm_y, pair ? tm_lo : tm_y, g);
}
