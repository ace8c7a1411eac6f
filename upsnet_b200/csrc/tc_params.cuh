// tc_params.cuh -- launch parameters and host helpers shared by the wgmma convolution kernels and the C-ABI dispatcher.
#pragma once
#include <cuda.h>   // CUtensorMap + enums only; the encoder is resolved at run time (no libcuda link dependency)
#include <cuda_runtime.h>
#include <cstdint>

namespace ups {

// Rows of each packed weight plane (hi, lo) of the tensor-core convs: Cout zero-padded to a whole number of N tiles.
inline int cout_pad(int Cout) { return Cout <= 32 ? 32 : (Cout + 63) / 64 * 64; }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled from the driver, looked up once; null when the driver does not have it
inline EncodeTiledFn tma_encoder() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qr = cudaDriverEntryPointSymbolNotFound;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess &&
        qr == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
    else
      (void)cudaGetLastError();
    tried = true;
  }
  return fn;
}

struct TcParams {
  const void* x;         // NHWC [N,H,W,Cin], fp32 or bf16 (x_bf16)
  const float* offset;   // NCHW fp32 [N,2*KHW,Ho,Wo] or null
  const float* mask;     // NCHW fp32 [N,KHW,Ho,Wo] or null
  const uint16_t* w_hi;  // bf16 [Cout_pad][KHW*Cin]
  const uint16_t* w_lo;  // bf16 residual plane (BF16X3) or null
  const float* bias; const void* residual; void* y;   // residual / y: fp32 or bf16 (y_bf16)
  int N, H, W, Cin, Cout, Cout_pad, kh, kw, sh, sw, ph, pw, dh, dw, Ho, Wo;
  int relu, out_nhwc, BN, stages, x3;
  int x_bf16, y_bf16;    // activation storage: 0 = fp32, 1 = bf16 (x / y+residual)
  int x_pair, y_pair;    // activation storage: hi/lo bf16 PAIRS, NHWC with 2*C channels ([0,C) = bf16(v), [C,2C) = bf16(v - hi));
                         // precision bf16x3 on bf16 storage: same bytes as fp32, but TMA / cp.async can feed the tensor core directly
  int sig_from;          // output channels >= sig_from get 1 / (1 + expf(-v)) (direct / per-lane epilogues only); -1 = none
  int pair_group;        // y_pair: channels are stored [hi G][lo G] per group of G channels (0 = Cout; TMA kernel only)
  int res_up2;           // residual is a half-resolution NHWC map read with nearest-neighbour 2x upsampling
  int no_tma;            // UPSNET_EPI_NO_TMA: force the cp.async gather kernel (A/B comparisons, tests)
  int tile_w, tile_h;    // deformable mode: pixel block of an M-tile (16x8 = all 128 rows; 8x8 / 8x4 leave rows unused)
  const int* n_dev;      // optional device-side image count (<= N): the TMA kernel skips the tiles of images >= *n_dev
};

size_t tc_packed_weight_bytes(int Cout, int Cin, int kh, int kw);
int tc_pack_weight(const float* w, int Cout, int Cin, int kh, int kw, void* packed, cudaStream_t stream);
bool tc_supported(int Cin, int kh, int kw, int dg);
int launch_igemm_tc(TcParams p, const void* packed, cudaStream_t stream);
// TMA-fed variant (igemm_tma.cu): returns UPSNET_E_UNSUPPORTED when the layer does not qualify
int launch_igemm_tma(const TcParams& p, const void* packed, cudaStream_t stream);

}  // namespace ups
