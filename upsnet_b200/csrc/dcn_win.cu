// dcn_win.cu -- fused deformable convolution (v1 / v2) on hi/lo bf16 PAIR activations with the bilinear corners
// gathered from a SHARED-MEMORY WINDOW instead of global memory (sm_90a).
//
// Reference semantics: operators/src/deform_conv_kernel.cu:89-118 (bilinear corner rule), :194-242 (im2col, the
// h > -1 && w > -1 && h < H && w < W test at :229), operators/functions/deform_conv.py:44-57 (im2col + torch.mm);
// v2 mask: operators/src/mod_deform_conv_kernel.cu.  Same arithmetic contract as igemm_tc_kernel<1,2> (igemm_tc.cu),
// which this kernel replaces for 3x3 / stride-1 layers on the pair stream: that kernel's gather is issue-bound -- a few
// hundred instructions per (pixel, tap, 8 channels), much of it 64-bit address arithmetic and unpacking around eight
// long-latency global loads.
//
// Here the K axis is ordered (16-channel sub-chunk, tap, channel): for one sub-chunk the nine taps x four corners of a
// 16 x 8-pixel tile touch one small window of the input -- (16 + 3 + offset range) x (8 + 3 + offset range) pixels x
// 16 channels x (hi, lo) -- which ONE TMA box pair stages in shared memory (32 x 20 pixels, 2 x 20 KB, double buffered).
// The 16 gather warps then read corners with LDS.128 at immediate offsets (+32 B = x+1, +960 B = y+1), blend (hi plane:
// fp32 FMAs, lo plane: packed bf16x2 HFMA2), re-split and store the A tile in the SWIZZLE_128B K-major layout
// wgmma consumes; weights (packed in the same K order by dcn_win_pack_weight) arrive by TMA.  Samples that fall
// outside the window (large offsets) are flagged in the per-tile sample table and gathered from global memory by the
// same thread, so the result never depends on the window size -- only the speed does.
//
// Two instantiations, chosen per launch (DwCfg below):
//   N tile 128 (semantic head, res3-5 DCN): 20 warps.  0-7 consumers (two warpgroups, tile rows 0-63 / 64-127, one
//     m64n128 fragment per thread; per K=16 slice three wgmma -- lo*hi, hi*lo, hi*hi), 8 weight TMA, 9 window TMA,
//     10-11 idle, 12-19 gather producers.  K = 32 per stage (SWIZZLE_64B), three stages.  The A tile is gathered once
//     per 128 output channels.
//   N tile 32 (small maps, Cout not a multiple of 128): 24 warps.  0-3 consumers (one warpgroup holding both m64n32
//     fragments), 4 weight TMA, 5 window TMA, 6-7 idle, 8-23 gather producers.  K = 64 per stage (SWIZZLE_128B), two
//     stages.
//   The TMA warps and the idle ones form a warpgroup that hands registers to the consumers (setmaxnreg, DwCfg).
// In both, a producer warp gathers two K=16 slices of 32 tile rows per k-block, and the producers form two groups that
// fill alternate k-blocks.  After the last k-block of a tile each consumer warpgroup stages its accumulators through
// shared memory (32 columns at a time) -> bias / ReLU -> hi/lo split -> NHWC pair stores, thread = tile pixel.
// Every output element sums the same K=16 slices in the same order in both instantiations.
// Roofline: tensor pipe (2*P*Cout*Cin*9 flop x 3 passes); per 64 K and SM the gather costs ~4 K warp instructions and
// 128 KB of shared-memory reads -- per 128 output channels at N = 128, per 32 at N = 32 -- see DESIGN.md section 4.
#include <cuda.h>
#include <cuda_bf16.h>

#include "common.cuh"
#include "tc_ptx.cuh"
#include "tc_params.cuh"

namespace ups {

constexpr int DW_BM = 128;            // pixels per M tile
constexpr int DW_WW = 32, DW_WH = 20; // window box in pixels; the row pitch (32 px = 1024 B) keeps bank = f(x) only
constexpr int DW_PLANE = DW_WW * DW_WH * 32;      // one plane (hi or lo) of a window: 16 channels x 2 B per pixel
constexpr int DW_WIN_BYTES = 2 * DW_PLANE;
constexpr int DW_WIN_BUFS = 2;        // window buffers: the next fill streams in while the current one is gathered
constexpr int DW_KHW = 9;
constexpr int DW_GROUPS = 2;          // producer groups: alternate k-blocks
constexpr int DW_EPI_PITCH = 36;      // floats per row of the accumulator staging buffer (32 columns + pad)
constexpr uint32_t DW_EPI_BYTES = DW_BM * DW_EPI_PITCH * 4;

// shared-memory map (byte offsets from the 1024-aligned base); the stages, windows and staging buffer follow (DwCfg)
constexpr uint32_t DW_OFF_BARS = 0;        // 18 mbarriers
constexpr uint32_t DW_OFF_STATS = 192;     // 2 x int[8]: min w, min h, max w, max h, sum w, sum h, count, -
constexpr uint32_t DW_OFF_ORG = 256;       // 2 x int4: window origin (w, h), image, -
constexpr uint32_t DW_OFF_TW = 512;        // float4 [9][128] corner weights
constexpr uint32_t DW_OFF_TP = DW_OFF_TW + DW_KHW * DW_BM * 16;   // int [9][128] window byte offset / outlier code
constexpr uint32_t DW_OFF_STAGES = DW_OFF_TP + DW_KHW * DW_BM * 4;   // 23552 = 23 * 1024
static_assert(DW_OFF_STAGES % 1024 == 0, "stage buffers need 1024-byte alignment (SWIZZLE_128B)");

// Per-instantiation geometry.  N tile 32: one consumer warpgroup holds both m64 fragments (2 x 16 floats) next to 16
// gather warps.  N tile 128: an m64n128 fragment is 64 floats per thread, so each tile half gets its own consumer
// warpgroup and the gather runs on 8 warps (16 gather warps would leave the consumers too few registers); its stages
// hold K = 32 so that three of them, two windows and the staging buffer fit in 227 KB of shared memory.
template <int BN> struct DwCfg {
  static constexpr int NCW = BN == 128 ? 2 : 1;                  // consumer warpgroups
  static constexpr int FRAGS = 2 / NCW;                          // m64 accumulator fragments per consumer thread
  static constexpr int BK = BN == 128 ? 32 : 64;                 // K elements per k-block
  static constexpr int SPK = BK / 16;                            // K=16 slices per k-block
  static constexpr int ROWB = BK * 2;                            // bytes of one A / B row in a stage (= swizzle span)
  static constexpr int CONSUMERS = 128 * NCW;
  // one warpgroup for the two TMA warps (and two idle warps), so that setmaxnreg can move its registers to the consumers
  static constexpr int WARP_TMAB = CONSUMERS / 32, WARP_TMAW = WARP_TMAB + 1, WARP_PROD0 = WARP_TMAB + 4;
  static constexpr int GROUP = 4 * (SPK / 2) * 32;                // producer threads per group: 4 row quadrants x SPK/2
  static constexpr int PRODUCERS = GROUP * DW_GROUPS;
  static constexpr int THREADS = WARP_PROD0 * 32 + PRODUCERS;     // 768 (N = 32), 640 (N = 128)
  // registers per thread: the launch budget (80 for 24 warps, 96 for 20: 16 K registers per SM sub-partition) stays
  // with the producers; the TMA warpgroup drops to REGS_TMA and the consumer warpgroups take what it frees.  setmaxnreg
  // moves registers inside the CTA's own allocation, so the warpgroup budgets must add up to what the launch gave.
  // ptxas -v: no spills in either instantiation (N = 128: 64 accumulators per consumer thread).
  static constexpr int WARPGROUPS = THREADS / 128;
  static constexpr int REGS_LAUNCH = 16384 / (32 * ((THREADS / 32 + 3) / 4)) / 8 * 8;
  static constexpr int REGS_TMA = 32, REGS_CONSUMER = 128;
  static_assert(NCW * REGS_CONSUMER + REGS_TMA + (PRODUCERS / 128) * REGS_LAUNCH <= WARPGROUPS * REGS_LAUNCH,
                "setmaxnreg budgets exceed the CTA's register allocation");
  static constexpr int TABLE_IT = (DW_KHW * DW_BM + PRODUCERS - 1) / PRODUCERS;   // sample-table entries per producer
  static constexpr uint32_t A_BYTES = 2 * DW_BM * ROWB;          // A stage: hi tile, lo tile (128 rows x BK bf16)
  static constexpr uint32_t B_BYTES = BN * ROWB;                 // one weight plane of a stage
  static constexpr uint32_t STAGE_BYTES = 2 * B_BYTES + A_BYTES;
  static_assert(STAGE_BYTES % 1024 == 0, "stages must keep the 1024-byte alignment of the swizzled tiles");
  // operand ring depth (A stages from the gather warps, B stages from TMA): as many as fit next to the tables, the two
  // windows and the staging buffer.  N = 32: 23 KB tables + 2 x 40 KB stages (3 do not fit) + 2 x 40 KB windows + 18 KB
  // staging; N = 128: 23 KB tables + 3 x 32 KB stages + 2 x 40 KB windows + 18 KB staging.
  static constexpr int STAGES = BN == 128 ? 3 : 2;
  static_assert(STAGES <= 3, "the barrier map holds three stages");
  static constexpr uint32_t OFF_WIN = DW_OFF_STAGES + STAGES * STAGE_BYTES;   // window buffers (1024-aligned)
  static constexpr uint32_t OFF_EPI = OFF_WIN + DW_WIN_BUFS * DW_WIN_BYTES;   // accumulator staging buffer
  static constexpr uint32_t SMEM = OFF_EPI + DW_EPI_BYTES + 1024;             // + alignment slack of the dynamic base
  static_assert(SMEM <= 227 * 1024, "shared memory exceeds 227 KB");
};
// 16-byte chunk j of A / B row r in a stage: SWIZZLE_128B (128-byte rows) or SWIZZLE_64B (64-byte rows)
template <int ROWB> __device__ __forceinline__ uint32_t dw_chunk(uint32_t j, uint32_t r) {
  return ROWB == 128 ? (j ^ (r & 7u)) : (j ^ ((r >> 1) & 3u));
}

struct DwParams {
  const void* x;          // pair NHWC [N,H,W,2*Cin] (outlier gathers)
  const float* offset;    // NCHW fp32 [N,18,Ho,Wo]
  const float* mask;      // NCHW fp32 [N,9,Ho,Wo] or null
  const float* bias;
  void* y;                // pair NHWC [N,Ho,Wo,2*Cout]
  int N, H, W, Cin, Cout, Cout_pad, Ho, Wo, ph, pw, dh, dw, relu, BN, tile_w, tile_h;
};

// p is __grid_constant__ so that each field is read from the parameter bank where it is used.  Passed as a plain value,
// nvcc 12.9 loads the whole struct into registers at kernel entry and keeps it live, and both instantiations spill.
template <int BN>
__global__ void __launch_bounds__(DwCfg<BN>::THREADS, 1)
dcn_win_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ DwParams p) {
  using C = DwCfg<BN>;
  constexpr int DW_PRODUCERS = C::PRODUCERS, DW_CONSUMERS = C::CONSUMERS;
  constexpr int DW_WARP_TMAB = C::WARP_TMAB, DW_WARP_TMAW = C::WARP_TMAW, DW_WARP_PROD0 = C::WARP_PROD0;
  constexpr int DW_BK = C::BK, SPK = C::SPK, ROWB = C::ROWB;
  extern __shared__ __align__(1024) uint8_t smem_dyn[];
  const uint32_t raw = smem_u32(smem_dyn);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* sm = smem_dyn + (base - raw);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t b_bytes = C::B_BYTES;
  const uint32_t stage_bytes = C::STAGE_BYTES;                              // weight tile (hi, lo planes), then the A tiles
  constexpr uint32_t NST = C::STAGES, NWB = DW_WIN_BUFS;
  const uint32_t win_base = base + C::OFF_WIN;
  float* stf = reinterpret_cast<float*>(sm + C::OFF_EPI);                   // accumulator staging
  // barriers
  const uint32_t bar_fa = base + DW_OFF_BARS;            // full_a[3]: the producer warps of one group (A stage written)
  const uint32_t bar_fb = bar_fa + 24;                   // full_b[3]: weight TMA (tx)
  const uint32_t bar_em = bar_fa + 48;                   // empty[3]: every consumer warp (its wgmmas have read A and B)
  const uint32_t bar_wf = bar_fa + 104;                  // win_full[2]: window TMA (tx)
  const uint32_t bar_we = bar_fa + 120;                  // win_empty[2]: every producer warp
  const uint32_t bar_og = bar_fa + 136;                  // org_full[2]: window origin of a tile published
  int* stats = reinterpret_cast<int*>(sm + DW_OFF_STATS);
  int4* org = reinterpret_cast<int4*>(sm + DW_OFF_ORG);
  float4* tw = reinterpret_cast<float4*>(sm + DW_OFF_TW);
  int* tp = reinterpret_cast<int*>(sm + DW_OFF_TP);

  const int HoWo = p.Ho * p.Wo;
  const int nsc = p.Cin / 16;                         // 16-channel sub-chunks = window fills per tile
  const int num_kb = nsc * DW_KHW / SPK;              // Cin % 64 == 0 -> integral
  const int n_tiles = p.Cout_pad / BN;
  const int TW = p.tile_w, TH = p.tile_h;
  const int tw_shift = TW == 16 ? 4 : 3;
  const int tiles_w = (p.Wo + TW - 1) / TW, tiles_h = (p.Ho + TH - 1) / TH;
  const long long num_tiles = (long long)p.N * tiles_w * tiles_h * n_tiles;

  if (warp == 0) {
    if (lane == 0) {
      for (int s = 0; s < C::STAGES; ++s) {
        mbar_init(bar_fa + 8 * s, C::GROUP / 32);
        mbar_init(bar_fb + 8 * s, 1);
        mbar_init(bar_em + 8 * s, DW_CONSUMERS / 32);
      }
      for (int s = 0; s < 2; ++s) {
        mbar_init(bar_wf + 8 * s, 1);
        mbar_init(bar_we + 8 * s, DW_PRODUCERS / 32);
        mbar_init(bar_og + 8 * s, 1);
      }
      fence_mbar_init();
      for (int i = 0; i < 2; ++i) {
        stats[i * 8 + 0] = 0x7fffffff; stats[i * 8 + 1] = 0x7fffffff;
        stats[i * 8 + 2] = -0x7fffffff; stats[i * 8 + 3] = -0x7fffffff;
        stats[i * 8 + 4] = 0; stats[i * 8 + 5] = 0; stats[i * 8 + 6] = 0; stats[i * 8 + 7] = 0;
      }
    }
    __syncwarp();
  }
  if (warp == DW_WARP_TMAB && lane == 0) prefetch_tmap(&tm_w);
  if (warp == DW_WARP_TMAW && lane == 0) prefetch_tmap(&tm_x);
  __syncthreads();

  if (warp >= DW_WARP_PROD0) {
    // =============================== GATHER PRODUCERS ===============================
    // A warp owns 32 rows of the A tile (quadrant = producer warp % 4), lane = row: the 32 lanes of an LDS.128 read one
    // (slice, 8-channel half) of 32 consecutive tile pixels.  The window is stored by
    // TMA with SWIZZLE_32B (16-byte chunk ^= address bit 7, i.e. pixel bit 2), so eight horizontally consecutive pixels of
    // one half occupy eight different 16-byte bank groups: a quarter-warp wavefront is conflict-free whenever its samples
    // stay on consecutive pixels of any rows (row pitch 1024 B).
    const int pt = tid - DW_WARP_PROD0 * 32;     // sample-table work is spread over all producer threads
    const int pw = warp - DW_WARP_PROD0;
    const int group = pw / (C::GROUP / 32);      // alternate k-blocks
    const int u = (pw >> 2) & (SPK / 2 - 1);     // which two of the k-block's slices this warp gathers
    const int quad = pw & 3;                     // A rows [32 quad, 32 quad + 32)
    const int r = quad * 32 + lane;              // A row = tile pixel
    const __nv_bfloat16* xh = reinterpret_cast<const __nv_bfloat16*>(p.x);
    uint32_t g0 = 0, wf0 = 0;                    // running k-block / window-fill counters at the start of the tile
    uint32_t wf_ready = 0;                       // window fills [0, wf_ready) have been observed complete by this thread
    uint32_t tile_it = 0;
    for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++tile_it) {
      const long long mt = tile / n_tiles;
      const int tx = (int)(mt % tiles_w), ty = (int)((mt / tiles_w) % tiles_h), n = (int)(mt / ((long long)tiles_w * tiles_h));
      const int par = (int)(tile_it & 1u);
      // ---- sample table, phase 1: every thread computes up to TABLE_IT (tap, pixel) entries in registers ----
      constexpr int TIT = C::TABLE_IT;
      float4 ewv[TIT];
      int ehl[TIT], ewl[TIT];
      bool evalid[TIT];
      int mnw = 0x7fffffff, mnh = 0x7fffffff, mxw = -0x7fffffff, mxh = -0x7fffffff, sw_ = 0, sh_ = 0, cnt = 0;
#pragma unroll
      for (int it = 0; it < TIT; ++it) {
        const int e = pt + it * DW_PRODUCERS;
        ewv[it] = make_float4(0.f, 0.f, 0.f, 0.f);
        ehl[it] = 0; ewl[it] = 0; evalid[it] = false;
        if (e < DW_KHW * DW_BM) {
          const int tap = e >> 7, rr = e & 127;
          const int ry = rr >> tw_shift;
          const int wo = tx * TW + (rr & (TW - 1)), ho = ty * TH + ry;
          if (ry < TH && wo < p.Wo && ho < p.Ho) {
            const int pp = ho * p.Wo + wo;
            const int ki = tap / 3, kj = tap - ki * 3;
            const float* offp = p.offset + ((size_t)n * 2 * DW_KHW + 2 * tap) * HoWo + pp;
            const float oh = __ldg(offp), ow = __ldg(offp + HoWo);
            const float h = (float)(ho - p.ph + ki * p.dh) + oh;
            const float w = (float)(wo - p.pw + kj * p.dw) + ow;
            if (h > -1.f && w > -1.f && h < (float)p.H && w < (float)p.W) {      // deform_conv_kernel.cu:229
              const int hl = (int)floorf(h), wl = (int)floorf(w), hh = hl + 1, wh = wl + 1;
              const float lh = h - hl, lw = w - wl, ch = 1.f - lh, cw = 1.f - lw;
              const bool t_ok = hl >= 0, b_ok = hh <= p.H - 1, l_ok = wl >= 0, r_ok = wh <= p.W - 1;
              float m = 1.f;
              if (p.mask) m = __ldg(p.mask + ((size_t)n * DW_KHW + tap) * HoWo + pp);
              ewv[it].x = (t_ok && l_ok) ? ch * cw * m : 0.f;
              ewv[it].y = (t_ok && r_ok) ? ch * lw * m : 0.f;
              ewv[it].z = (b_ok && l_ok) ? lh * cw * m : 0.f;
              ewv[it].w = (b_ok && r_ok) ? lh * lw * m : 0.f;
              ehl[it] = hl; ewl[it] = wl; evalid[it] = true;
              mnw = min(mnw, wl); mxw = max(mxw, wl + 1); mnh = min(mnh, hl); mxh = max(mxh, hl + 1);
              sw_ += wl; sh_ += hl; ++cnt;
            }
          }
        }
      }
      mnw = __reduce_min_sync(0xffffffffu, mnw); mnh = __reduce_min_sync(0xffffffffu, mnh);
      mxw = __reduce_max_sync(0xffffffffu, mxw); mxh = __reduce_max_sync(0xffffffffu, mxh);
      sw_ = __reduce_add_sync(0xffffffffu, sw_); sh_ = __reduce_add_sync(0xffffffffu, sh_);
      cnt = __reduce_add_sync(0xffffffffu, cnt);
      if (lane == 0 && cnt > 0) {
        int* st = stats + par * 8;
        atomicMin(st + 0, mnw); atomicMin(st + 1, mnh); atomicMax(st + 2, mxw); atomicMax(st + 3, mxh);
        atomicAdd(st + 4, sw_); atomicAdd(st + 5, sh_); atomicAdd(st + 6, cnt);
      }
      named_bar<1, DW_PRODUCERS>();      // (B) statistics complete; every producer has also finished the previous tile's gather
      // ---- window origin (same integer arithmetic in every thread), table phase 2 ----
      int ox = 0, oy = 0;
      {
        const int* st = stats + par * 8;
        const int c = st[6];
        if (c > 0) {
          const int a = st[0], b = st[1], cc = st[2], d = st[3];
          // the bounding box of all corners fits: start the window there; otherwise centre it on the mean sample
          ox = (cc - a + 1 <= DW_WW) ? a : (int)floorf((float)st[4] / (float)c + 1.0f) - DW_WW / 2;
          oy = (d - b + 1 <= DW_WH) ? b : (int)floorf((float)st[5] / (float)c + 1.0f) - DW_WH / 2;
        }
      }
#pragma unroll
      for (int it = 0; it < TIT; ++it) {
        const int e = pt + it * DW_PRODUCERS;
        if (e < DW_KHW * DW_BM) {
          int code = 0;
          if (evalid[it]) {
            const int dx = ewl[it] - ox, dy = ehl[it] - oy;
            if (dx >= 0 && dx + 1 < DW_WW && dy >= 0 && dy + 1 < DW_WH) code = (dy * DW_WW + dx) * 32;
            else code = (int)(0x80000000u | ((uint32_t)(ehl[it] + 1) << 15) | (uint32_t)(ewl[it] + 1));   // outlier: global gather
          }
          tw[e] = ewv[it];
          tp[e] = code;
        }
      }
      if (pt == 0) {
        org[par] = make_int4(ox, oy, n, 0);
        int* so = stats + (par ^ 1) * 8;      // reset the other slot for the next tile (last read before barrier B of this tile)
        so[0] = 0x7fffffff; so[1] = 0x7fffffff; so[2] = -0x7fffffff; so[3] = -0x7fffffff; so[4] = 0; so[5] = 0; so[6] = 0;
        mbar_arrive(bar_og + 8 * par);        // release: the window TMA thread may read the origin
      }
      named_bar<1, DW_PRODUCERS>();      // (C) table visible
      const __nv_bfloat16* ximg = xh + (size_t)n * p.H * p.W * (size_t)(2 * p.Cin);

      int rel = 0;            // sub-chunks of this tile this WARP has released
      for (int kb = (int)((uint32_t)(group - (int)g0) & 1u); kb < num_kb; kb += DW_GROUPS) {
        const uint32_t g = g0 + (uint32_t)kb;
        const uint32_t s = g % NST, it = g / NST;
        mbar_wait(bar_em + 8 * s, (it & 1u) ^ 1u);
        // A stage s: hi tile then lo tile, row r = ROWB bytes, 16-byte chunk j of K at dw_chunk(j, r)
        const uint32_t a_row = base + DW_OFF_STAGES + s * stage_bytes + 2 * b_bytes + (uint32_t)r * (uint32_t)ROWB;
#pragma unroll 1
        for (int pass = 0; pass < 4; ++pass) {
          const int sl = 2 * u + (pass >> 1), half = pass & 1;
          const int q = kb * SPK + sl;                  // slice index: (sub-chunk, tap)
          const int sc = q / DW_KHW, tap = q - sc * DW_KHW;
          const uint32_t wf = wf0 + (uint32_t)sc;
          if (wf >= wf_ready) {                         // first touch of this window fill
            mbar_wait(bar_wf + 8 * (wf % NWB), (wf / NWB) & 1u);
            wf_ready = wf + 1;
          }
          const uint32_t wbuf = win_base + (wf % NWB) * (uint32_t)DW_WIN_BYTES;
          const int code = tp[tap * DW_BM + r];
          const uint32_t a_off = dw_chunk<ROWB>((uint32_t)(sl * 2 + half), (uint32_t)r) << 4;   // K elements 16 sl + 8 half ..
          const float4 wv = tw[tap * DW_BM + r];
          uint4 hc[4], lc[4];
          if (code >= 0) {
            // SWIZZLE_32B: the 16-byte chunk of a pixel sits at (half ^ bit 7 of the pixel's byte offset)
            const uint32_t cl = (uint32_t)code, cr = cl + 32u;
            const uint32_t al = wbuf + cl + ((((cl >> 7) & 1u) ^ (uint32_t)half) << 4);
            const uint32_t ar = wbuf + cr + ((((cr >> 7) & 1u) ^ (uint32_t)half) << 4);
            hc[0] = lds128(al); hc[1] = lds128(ar); hc[2] = lds128(al + DW_WW * 32); hc[3] = lds128(ar + DW_WW * 32);
            lc[0] = lds128(al + DW_PLANE); lc[1] = lds128(ar + DW_PLANE);
            lc[2] = lds128(al + DW_PLANE + DW_WW * 32); lc[3] = lds128(ar + DW_PLANE + DW_WW * 32);
          } else {
            // outlier sample: the four corners come from global memory (clamped addresses; invalid corners carry weight 0)
            const int hl = (int)(((uint32_t)code >> 15) & 0xffffu) - 1, wl = (int)((uint32_t)code & 0x7fffu) - 1;
            const int h0 = max(hl, 0), h1 = min(hl + 1, p.H - 1), w0 = max(wl, 0), w1 = min(wl + 1, p.W - 1);
            const size_t pc = (size_t)(2 * p.Cin);
            const int cg = sc * 16 + half * 8;            // first channel of this pass's 8-channel vector
            const __nv_bfloat16* b00 = ximg + ((size_t)h0 * p.W + w0) * pc + cg;
            const __nv_bfloat16* b01 = ximg + ((size_t)h0 * p.W + w1) * pc + cg;
            const __nv_bfloat16* b10 = ximg + ((size_t)h1 * p.W + w0) * pc + cg;
            const __nv_bfloat16* b11 = ximg + ((size_t)h1 * p.W + w1) * pc + cg;
            hc[0] = __ldg(reinterpret_cast<const uint4*>(b00)); lc[0] = __ldg(reinterpret_cast<const uint4*>(b00 + p.Cin));
            hc[1] = __ldg(reinterpret_cast<const uint4*>(b01)); lc[1] = __ldg(reinterpret_cast<const uint4*>(b01 + p.Cin));
            hc[2] = __ldg(reinterpret_cast<const uint4*>(b10)); lc[2] = __ldg(reinterpret_cast<const uint4*>(b10 + p.Cin));
            hc[3] = __ldg(reinterpret_cast<const uint4*>(b11)); lc[3] = __ldg(reinterpret_cast<const uint4*>(b11 + p.Cin));
          }
          // blend and split again: the arithmetic of the gather kernel's pair path (igemm_tc.cu), shared through pair.cuh
          uint4 ohi, olo;
          pair_blend8(wv, hc, lc, ohi, olo);
          sts128(a_row + a_off, ohi);
          sts128(a_row + DW_BM * ROWB + a_off, olo);
        }
        fence_proxy_async();    // generic-proxy stores -> visible to wgmma (async proxy)
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(bar_fa + 8 * s);
          // window buffers this warp will not read again: its next k-block (kb + 2) starts at slice SPK * (kb + 2)
          while (rel < nsc && DW_KHW * (rel + 1) <= SPK * (kb + DW_GROUPS)) {
            mbar_arrive(bar_we + 8 * ((wf0 + (uint32_t)rel) % NWB));
            ++rel;
          }
        }
        rel = __shfl_sync(0xffffffffu, rel, 0);
      }
      if (lane == 0) {
        while (rel < nsc) { mbar_arrive(bar_we + 8 * ((wf0 + (uint32_t)rel) % NWB)); ++rel; }
      }
      __syncwarp();
      g0 += (uint32_t)num_kb;
      wf0 += (uint32_t)nsc;
    }
  } else if (warp >= DW_WARP_TMAB) {
    // The TMA warpgroup (weight TMA, window TMA, two idle warps) keeps a minimal register budget so that the consumer
    // warpgroups can raise theirs.
    setmaxnreg_dec<C::REGS_TMA>();
    if (warp == DW_WARP_TMAW && lane == 0) {
    // =============================== WINDOW TMA ===============================
      uint32_t wf = 0, ti = 0;
      for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++ti) {
        const uint32_t par = ti & 1u;
        mbar_wait(bar_og + 8 * par, (ti >> 1) & 1u);
        const volatile int* ov = reinterpret_cast<const volatile int*>(&org[par]);
        const int4 o = make_int4(ov[0], ov[1], ov[2], 0);
        for (int f = 0; f < nsc; ++f, ++wf) {
          const uint32_t b = wf % NWB;
          mbar_wait(bar_we + 8 * b, ((wf / NWB) & 1u) ^ 1u);
          mbar_arrive_expect_tx(bar_wf + 8 * b, (uint32_t)DW_WIN_BYTES);
          const uint32_t dst = win_base + b * (uint32_t)DW_WIN_BYTES;
          tma_load_4d(dst, &tm_x, bar_wf + 8 * b, f * 16, o.x, o.y, o.z);
          tma_load_4d(dst + (uint32_t)DW_PLANE, &tm_x, bar_wf + 8 * b, p.Cin + f * 16, o.x, o.y, o.z);
        }
      }
    } else if (warp == DW_WARP_TMAB && lane == 0) {
      // =============================== WEIGHT TMA ===============================
      uint32_t g = 0;
      for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int n0 = (int)(tile % n_tiles) * BN;
        for (int kb = 0; kb < num_kb; ++kb, ++g) {
          const uint32_t s = g % NST, it = g / NST;
          mbar_wait(bar_em + 8 * s, (it & 1u) ^ 1u);
          const uint32_t stage = base + DW_OFF_STAGES + s * stage_bytes;
          mbar_arrive_expect_tx(bar_fb + 8 * s, 2 * b_bytes);
          tma_load_2d(stage, &tm_w, bar_fb + 8 * s, kb * DW_BK, n0);
          tma_load_2d(stage + b_bytes, &tm_w, bar_fb + 8 * s, kb * DW_BK, p.Cout_pad + n0);
        }
      }
    }
    __syncwarp();
  } else {
    // =============================== CONSUMERS (warpgroups 0 .. NCW-1) ===============================
    setmaxnreg_inc<C::REGS_CONSUMER>();
    // Warpgroup wg owns m64 fragment f (tile rows [64 (wg FRAGS + f), +64)) for f < FRAGS.
    constexpr int FRAGS = C::FRAGS;
    const int wg = warp >> 2;
    const uint32_t dhi = ROWB == 128 ? wg_desc_hi(8 * ROWB) : wg_desc_hi_sw64(8 * ROWB);
    float d[FRAGS][BN / 2];
    constexpr uint32_t h16 = 64u * ROWB / 16u;      // the next 64 tile rows: 64 rows of ROWB bytes further
    __nv_bfloat16* yb = reinterpret_cast<__nv_bfloat16*>(p.y);
    uint32_t s = 0, ph = 0;
    for (long long tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const long long mt = tile / n_tiles;
      const int n0 = (int)(tile % n_tiles) * BN;
      const int tx = (int)(mt % tiles_w), ty = (int)((mt / tiles_w) % tiles_h), n = (int)(mt / ((long long)tiles_w * tiles_h));
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(bar_fb + 8 * s, ph);
        mbar_wait(bar_fa + 8 * s, ph);
        const uint32_t st0 = base + DW_OFF_STAGES + s * stage_bytes;
        const uint32_t b_hi = wg_desc_lo(st0), b_lo = wg_desc_lo(st0 + b_bytes);
        const uint32_t a_hi = wg_desc_lo(st0 + 2 * b_bytes) + (uint32_t)(wg * FRAGS) * h16;
        const uint32_t a_lo = wg_desc_lo(st0 + 2 * b_bytes + DW_BM * ROWB) + (uint32_t)(wg * FRAGS) * h16;
        wgmma_fence();
#pragma unroll
        for (uint32_t k = 0; k < SPK; ++k) {
          const uint32_t acc = (kb | k) ? 1u : 0u;
          const uint64_t bh = wg_desc(b_hi + 2 * k, dhi), bl = wg_desc(b_lo + 2 * k, dhi);
#pragma unroll
          for (int f = 0; f < FRAGS; ++f) Wgmma<BN>::mma(d[f], wg_desc(a_lo + f * h16 + 2 * k, dhi), bh, acc);
#pragma unroll
          for (int f = 0; f < FRAGS; ++f) Wgmma<BN>::mma(d[f], wg_desc(a_hi + f * h16 + 2 * k, dhi), bl, 1u);
#pragma unroll
          for (int f = 0; f < FRAGS; ++f) Wgmma<BN>::mma(d[f], wg_desc(a_hi + f * h16 + 2 * k, dhi), bh, 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();                                // the previous k-block's wgmmas have read their stage
#pragma unroll
        for (int f = 0; f < FRAGS; ++f) wgmma_fence_acc(d[f]);
        if (prev >= 0 && lane == 0) mbar_arrive(bar_em + 8 * prev);
        prev = (int)s;
        if (++s == NST) { s = 0; ph ^= 1u; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int f = 0; f < FRAGS; ++f) wgmma_fence_acc(d[f]);
      if (prev >= 0 && lane == 0) mbar_arrive(bar_em + 8 * prev);

      // ---- epilogue per warpgroup: 32 accumulator columns at a time through shared memory, thread = tile pixel ----
      // One warpgroup: thread t has tile row t and both 16-column halves of a chunk.  Two: warpgroup wg has rows
      // [64 wg, 64 wg + 64), thread t of it row 64 wg + t % 64 and the chunk's 16-column half t / 64.
      const int t = tid & 127;
      const int m = FRAGS == 2 ? t : 64 * wg + (t & 63);
      const int csub = FRAGS == 2 ? 0 : 16 * (t >> 6), cstep = FRAGS == 2 ? 16 : 32;
      const int ry = m >> tw_shift;
      const int wo = tx * TW + (m & (TW - 1)), ho = ty * TH + ry;
      const bool row_ok = ry < TH && wo < p.Wo && ho < p.Ho;
      __nv_bfloat16* yp = yb + (((size_t)n * p.Ho + ho) * p.Wo + wo) * (size_t)(2 * p.Cout);
      const uint32_t trow = smem_u32(stf + (size_t)m * DW_EPI_PITCH);
      for (int c32 = 0; c32 < BN; c32 += 32) {
        if (n0 + c32 >= p.Cout) break;                 // zero-padded weight rows (CTA-uniform)
        named_bar(2 + wg, 128);                        // the previous chunk has been read
#pragma unroll
        for (int c = 0; c < BN; c += 32)
          if (c == c32) {
#pragma unroll
            for (int f = 0; f < FRAGS; ++f) acc_stage<BN, 32>(d[f], stf, DW_EPI_PITCH, 64 * (wg * FRAGS + f), c);
          }
        named_bar(2 + wg, 128);
        for (int cb = c32 + csub; cb < c32 + 32 && cb < BN; cb += cstep) {
          if (n0 + cb >= p.Cout) break;
          uint32_t rr[16];
          acc_ld16(trow + (uint32_t)(cb - c32) * 4u, rr);
          if (!row_ok) continue;
          const int co = n0 + cb;
          float o[16];
#pragma unroll
          for (int e = 0; e < 16; ++e) o[e] = __uint_as_float(rr[e]);
          if (p.bias) {
            if (co + 16 <= p.Cout) {
#pragma unroll
              for (int e4 = 0; e4 < 4; ++e4) {
                const float4 bv = __ldg(reinterpret_cast<const float4*>(p.bias + co) + e4);
                o[4 * e4] += bv.x; o[4 * e4 + 1] += bv.y; o[4 * e4 + 2] += bv.z; o[4 * e4 + 3] += bv.w;
              }
            } else {
#pragma unroll
              for (int e = 0; e < 16; ++e)
                if (co + e < p.Cout) o[e] += __ldg(p.bias + co + e);
            }
          }
          if (p.relu) {
#pragma unroll
            for (int e = 0; e < 16; ++e) o[e] = fmaxf(o[e], 0.f);
          }
          uint32_t hw[8], lw[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) split_pair2(o[2 * e], o[2 * e + 1], hw[e], lw[e]);
          uint4* dh_ = reinterpret_cast<uint4*>(yp + co);
          uint4* dl_ = reinterpret_cast<uint4*>(yp + p.Cout + co);
          dh_[0] = make_uint4(hw[0], hw[1], hw[2], hw[3]); dh_[1] = make_uint4(hw[4], hw[5], hw[6], hw[7]);
          dl_[0] = make_uint4(lw[0], lw[1], lw[2], lw[3]); dl_[1] = make_uint4(lw[4], lw[5], lw[6], lw[7]);
        }
      }
    }
  }
}

// ----------------------------------------------------------------------------------------------
// weight pre-pack: fp32 [Cout,Cin,3,3] -> bf16 hi / lo planes [Cout_pad][K], k = (c / 16) * 144 + tap * 16 + c % 16
// ----------------------------------------------------------------------------------------------
__global__ void dcn_win_pack_kernel(const float* __restrict__ w, int Cout, int Cin, int Cout_pad, int K,
                                    uint16_t* __restrict__ hi, uint16_t* __restrict__ lo) {
  const size_t total = (size_t)Cout_pad * K;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int kk = (int)(i % (size_t)K), co = (int)(i / (size_t)K);
    const int sc = kk / (16 * DW_KHW), rem = kk - sc * 16 * DW_KHW, tap = rem >> 4, c = sc * 16 + (rem & 15);
    const float v = co < Cout ? w[((size_t)co * Cin + c) * DW_KHW + tap] : 0.f;
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    hi[i] = *reinterpret_cast<const uint16_t*>(&h);
    lo[i] = *reinterpret_cast<const uint16_t*>(&l);
  }
}

// packing / kernel: any Cout (rows are zero-padded); the pair NHWC epilogue additionally needs Cout % 16 == 0
static bool dw_supported(int Cin, int Cout, int kh, int kw) {
  return kh == 3 && kw == 3 && Cin % 64 == 0 && Cin >= 64 && Cout >= 1;
}

}  // namespace ups

extern "C" int upsnet_dcn_packed_weight_bytes(int Cout, int Cin, int kh, int kw, size_t* bytes) {
  if (!bytes || Cout <= 0 || Cin <= 0) return UPSNET_E_BADARG;
  if (!ups::dw_supported(Cin, Cout, kh, kw)) return UPSNET_E_UNSUPPORTED;
  *bytes = (size_t)2 * ups::cout_pad(Cout) * (size_t)(9 * Cin) * sizeof(uint16_t);
  return 0;
}

extern "C" int upsnet_dcn_pack_weight(const float* weight, int Cout, int Cin, int kh, int kw, void* packed, void* stream) {
  if (!weight || !packed || Cout <= 0 || Cin <= 0) return UPSNET_E_BADARG;
  if (!ups::dw_supported(Cin, Cout, kh, kw)) return UPSNET_E_UNSUPPORTED;
  const int Cout_pad = ups::cout_pad(Cout), K = 9 * Cin;
  uint16_t* hi = reinterpret_cast<uint16_t*>(packed);
  uint16_t* lo = hi + (size_t)Cout_pad * K;
  const size_t total = (size_t)Cout_pad * K;
  int blocks = (int)((total + 255) / 256);
  if (blocks > ups::kNumSMs * 16) blocks = ups::kNumSMs * 16;
  ups::dcn_win_pack_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(weight, Cout, Cin, Cout_pad, K, hi, lo);
  UPS_CHECK_LAUNCH();
  return 0;
}

// N tile of the next launches: 0 = chosen per launch (below), 32 or 128 = that N tile wherever it applies (128 needs
// Cout_pad % 128 == 0).  For tests and tuning: lets one process compare both instantiations.
static int g_dw_force_bn = 0;

extern "C" int upsnet_dcn_set_tile_n(int bn) {
  if (bn != 0 && bn != 32 && bn != 128) return UPSNET_E_BADARG;
  g_dw_force_bn = bn;
  return 0;
}

extern "C" int upsnet_dcn_pair_forward(const void* x_pair, const float* offset, const float* mask, const void* packed,
                                       const float* bias, void* y_pair, int N, int H, int W, int Cin, int Cout, int kh,
                                       int kw, int pad_h, int pad_w, int dil_h, int dil_w, int epi_flags, void* stream) {
  using namespace ups;
  if (!x_pair || !offset || !packed || !y_pair) return UPSNET_E_BADARG;
  if (N <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0 || pad_h < 0 || pad_w < 0 || dil_h <= 0 || dil_w <= 0) return UPSNET_E_BADARG;
  if (!dw_supported(Cin, Cout, kh, kw)) return UPSNET_E_UNSUPPORTED;
  if ((Cout % 16) != 0) return UPSNET_E_UNSUPPORTED;
  if (H >= 32767 || W >= 32767) return UPSNET_E_UNSUPPORTED;                 // outlier code packs (h, w) into 16 + 15 bits
  if ((((uintptr_t)x_pair) & 15) || (((uintptr_t)packed) & 15) || (((uintptr_t)y_pair) & 15) || (bias && (((uintptr_t)bias) & 15)))
    return UPSNET_E_UNSUPPORTED;
  DwParams p{};
  p.x = x_pair; p.offset = offset; p.mask = mask; p.bias = bias; p.y = y_pair;
  p.N = N; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout; p.Cout_pad = cout_pad(Cout);
  p.ph = pad_h; p.pw = pad_w; p.dh = dil_h; p.dw = dil_w;
  p.Ho = conv_out_size(H, pad_h, dil_h, 3, 1);
  p.Wo = conv_out_size(W, pad_w, dil_w, 3, 1);
  if (p.Ho <= 0 || p.Wo <= 0) return UPSNET_E_BADARG;
  p.relu = (epi_flags & UPSNET_EPI_RELU) ? 1 : 0;
  const int sms = num_sms();
  p.tile_w = 16; p.tile_h = 8;
  auto dtiles = [&]() { return (long long)p.N * ((p.Wo + p.tile_w - 1) / p.tile_w) * ((p.Ho + p.tile_h - 1) / p.tile_h) * (p.Cout_pad / p.BN); };
  // N tile: 128 (A tile gathered once per 128 output channels) when Cout_pad allows it and there are at least sms / 4
  // of its 16 x 8-pixel tiles; otherwise 32, whose smaller pixel blocks (below) spread tiny maps over more SMs.  Measured
  // on H100 SXM (400 W), 256 -> 128 channels: 64 x 128 map (64 tiles) 0.128 ms at N = 128 vs 0.221 ms at N = 32;
  // 32 x 64 map (16 tiles) 0.138 vs 0.115 ms.
  p.BN = 128;
  const bool wide_ok = p.Cout_pad % 128 == 0;
  const bool wide = wide_ok && (g_dw_force_bn == 128 || (g_dw_force_bn == 0 && dtiles() >= sms / 4));
  if (!wide) p.BN = 32;
  // few tiles (coarse pyramid levels): smaller pixel blocks -> more CTAs share the serial k-block chain
  if (!wide && dtiles() < sms / 2) { p.tile_w = 8; p.tile_h = 8; }
  if (!wide && dtiles() < sms / 2) { p.tile_h = 4; }
  const long long num_tiles = dtiles();
  if (num_tiles <= 0) return 0;
  const int bk = wide ? DwCfg<128>::BK : DwCfg<32>::BK;
  const size_t smem = wide ? DwCfg<128>::SMEM : DwCfg<32>::SMEM;
  EncodeTiledFn enc = tma_encoder();
  if (!enc) return UPSNET_E_UNSUPPORTED;
  CUtensorMap tm_x, tm_w;
  {
    const cuuint64_t dx[4] = {(cuuint64_t)(2 * Cin), (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    const cuuint64_t sx[3] = {(cuuint64_t)(2 * Cin) * 2, (cuuint64_t)W * (2 * Cin) * 2, (cuuint64_t)H * W * (2 * Cin) * 2};
    const cuuint32_t bx[4] = {16, DW_WW, DW_WH, 1};
    const cuuint32_t es[4] = {1, 1, 1, 1};
    if (enc(&tm_x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(x_pair), dx, sx, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_32B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return UPSNET_E_UNSUPPORTED;
    // weight box: BK x BN, rows of BK bf16 in the swizzle the stage's wgmma descriptors expect
    const cuuint64_t dwt[2] = {(cuuint64_t)(9 * Cin), (cuuint64_t)(2 * p.Cout_pad)};
    const cuuint64_t sw[1] = {(cuuint64_t)(9 * Cin) * 2};
    const cuuint32_t bw[2] = {(cuuint32_t)bk, (cuuint32_t)p.BN};
    if (enc(&tm_w, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(packed), dwt, sw, bw, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
            bk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return UPSNET_E_UNSUPPORTED;
  }
  static PerDeviceOnce configured;
  if (configured.need()) {
    UPS_CUDA(cudaFuncSetAttribute(dcn_win_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    UPS_CUDA(cudaFuncSetAttribute(dcn_win_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  }
  dim3 grid((unsigned)(num_tiles < sms ? num_tiles : sms));
  if (wide)
    dcn_win_kernel<128><<<grid, DwCfg<128>::THREADS, smem, (cudaStream_t)stream>>>(tm_x, tm_w, p);
  else
    dcn_win_kernel<32><<<grid, DwCfg<32>::THREADS, smem, (cudaStream_t)stream>>>(tm_x, tm_w, p);
  UPS_CHECK_LAUNCH();
  return 0;
}
