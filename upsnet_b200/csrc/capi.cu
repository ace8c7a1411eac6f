// capi.cu -- convolution / deformable-convolution entry points of the C ABI and dispatch
// between the fp32 CUDA-core tiles (igemm_simt.cu) and the wgmma tensor-core tiles
// (igemm_tc.cu).  See include/upsnet_b200.h for the contract of every symbol.
#include "common.cuh"
#include "tc_params.cuh"

namespace ups {
struct ConvParams {
  const float* x; const float* offset; const float* mask; const float* weight;
  const float* bias; const float* residual; float* y;
  int N, Cin, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, dg, Ho, Wo, relu;
};
int launch_igemm_simt(const ConvParams& p, cudaStream_t stream);

}  // namespace ups

extern "C" int upsnet_version(int* n_sm) {
  if (n_sm) {
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) == cudaSuccess &&
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess)
      *n_sm = sms;
    else
      *n_sm = -1;
  }
  return 90;
}

static int conv_common(const float* x, const float* offset, const float* mask, const float* weight,
                       const float* bias, const float* residual, float* y, int N, int Cin, int H,
                       int W, int Cout, int kh, int kw, int sh, int sw, int ph, int pw, int dh,
                       int dw, int dg, int epi_flags, int precision, void* stream) {
  if (!x || !weight || !y) return UPSNET_E_BADARG;
  if (N <= 0 || Cin <= 0 || H <= 0 || W <= 0 || Cout <= 0 || kh <= 0 || kw <= 0 || sh <= 0 ||
      sw <= 0 || ph < 0 || pw < 0 || dh <= 0 || dw <= 0 || dg <= 0 || Cin % dg != 0)
    return UPSNET_E_BADARG;
  ups::ConvParams p;
  p.x = x; p.offset = offset; p.mask = mask; p.weight = weight; p.bias = bias;
  p.residual = residual; p.y = y;
  p.N = N; p.Cin = Cin; p.H = H; p.W = W; p.Cout = Cout; p.kh = kh; p.kw = kw; p.sh = sh;
  p.sw = sw; p.ph = ph; p.pw = pw; p.dh = dh; p.dw = dw; p.dg = dg;
  p.Ho = ups::conv_out_size(H, ph, dh, kh, sh);
  p.Wo = ups::conv_out_size(W, pw, dw, kw, sw);
  p.relu = (epi_flags & UPSNET_EPI_RELU) ? 1 : 0;
  if (p.Ho <= 0 || p.Wo <= 0) return UPSNET_E_BADARG;
  if ((size_t)Cin * H * W >= (1ull << 31)) return UPSNET_E_UNSUPPORTED;  // int32 plane offsets
  switch (precision) {
    case UPSNET_PREC_FP32_SIMT:
      return ups::launch_igemm_simt(p, (cudaStream_t)stream);
    default:
      return UPSNET_E_UNSUPPORTED;
  }
}

extern "C" int upsnet_dcn_forward(const float* x, const float* offset, const float* mask,
                                  const float* weight, const float* bias, float* y, int N, int Cin,
                                  int H, int W, int Cout, int kh, int kw, int stride_h,
                                  int stride_w, int pad_h, int pad_w, int dil_h, int dil_w,
                                  int deformable_groups, int epi_flags, int precision,
                                  void* stream) {
  if (!offset) return UPSNET_E_BADARG;
  return conv_common(x, offset, mask, weight, bias, nullptr, y, N, Cin, H, W, Cout, kh, kw,
                     stride_h, stride_w, pad_h, pad_w, dil_h, dil_w, deformable_groups, epi_flags,
                     precision, stream);
}

extern "C" int upsnet_conv2d_forward(const float* x, const float* weight, const float* bias,
                                     const float* residual, float* y, int N, int Cin, int H, int W,
                                     int Cout, int kh, int kw, int stride_h, int stride_w,
                                     int pad_h, int pad_w, int dil_h, int dil_w, int epi_flags,
                                     int precision, void* stream) {
  return conv_common(x, nullptr, nullptr, weight, bias, residual, y, N, Cin, H, W, Cout, kh, kw,
                     stride_h, stride_w, pad_h, pad_w, dil_h, dil_w, 1, epi_flags, precision,
                     stream);
}

extern "C" int upsnet_igemm_packed_weight_bytes(int Cout, int Cin, int kh, int kw, size_t* bytes) {
  if (!bytes || Cout <= 0 || Cin <= 0 || kh <= 0 || kw <= 0) return UPSNET_E_BADARG;
  if (!ups::tc_supported(Cin, kh, kw, 1)) return UPSNET_E_UNSUPPORTED;
  *bytes = ups::tc_packed_weight_bytes(Cout, Cin, kh, kw);
  return 0;
}

extern "C" int upsnet_igemm_pack_weight(const float* weight, int Cout, int Cin, int kh, int kw,
                                        void* packed, void* stream) {
  if (!weight || !packed || Cout <= 0 || Cin <= 0 || kh <= 0 || kw <= 0) return UPSNET_E_BADARG;
  if (!ups::tc_supported(Cin, kh, kw, 1)) return UPSNET_E_UNSUPPORTED;
  return ups::tc_pack_weight(weight, Cout, Cin, kh, kw, packed, (cudaStream_t)stream);
}

extern "C" int upsnet_igemm_forward(const void* x_nhwc, const float* offset, const float* mask,
                                    const void* packed, const float* bias, const void* residual,
                                    void* y, int N, int H, int W, int Cin, int Cout, int kh, int kw,
                                    int stride_h, int stride_w, int pad_h, int pad_w, int dil_h,
                                    int dil_w, int out_layout, int x_dtype, int y_dtype, int epi_flags,
                                    int precision, const int* n_dev, void* stream) {
  if (!x_nhwc || !packed || !y) return UPSNET_E_BADARG;
  if (N <= 0 || Cin <= 0 || H <= 0 || W <= 0 || Cout <= 0 || kh <= 0 || kw <= 0 || stride_h <= 0 ||
      stride_w <= 0 || pad_h < 0 || pad_w < 0 || dil_h <= 0 || dil_w <= 0)
    return UPSNET_E_BADARG;
  if (precision != UPSNET_PREC_BF16X3 && precision != UPSNET_PREC_BF16) return UPSNET_E_BADARG;
  if (out_layout != UPSNET_LAYOUT_NCHW && out_layout != UPSNET_LAYOUT_NHWC) return UPSNET_E_BADARG;
  if (mask && !offset) return UPSNET_E_BADARG;
  if ((size_t)H * W >= (1ull << 31)) return UPSNET_E_UNSUPPORTED;
  ups::TcParams p{};
  p.x = x_nhwc; p.offset = offset; p.mask = mask; p.bias = bias; p.residual = residual; p.y = y;
  p.n_dev = n_dev;
  p.N = N; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout; p.kh = kh; p.kw = kw; p.sh = stride_h;
  p.sw = stride_w; p.ph = pad_h; p.pw = pad_w; p.dh = dil_h; p.dw = dil_w;
  p.Ho = ups::conv_out_size(H, pad_h, dil_h, kh, stride_h);
  p.Wo = ups::conv_out_size(W, pad_w, dil_w, kw, stride_w);
  if (p.Ho <= 0 || p.Wo <= 0) return UPSNET_E_BADARG;
  p.relu = (epi_flags & UPSNET_EPI_RELU) ? 1 : 0;
  p.out_nhwc = out_layout == UPSNET_LAYOUT_NHWC;
  p.res_up2 = (epi_flags & UPSNET_EPI_RES_UP2) ? 1 : 0;
  p.no_tma = (epi_flags & UPSNET_EPI_NO_TMA) ? 1 : 0;
  if (p.res_up2 && (!residual || !p.out_nhwc || (p.Ho & 1) || (p.Wo & 1))) return UPSNET_E_BADARG;
  p.x3 = precision == UPSNET_PREC_BF16X3;
  if (x_dtype < UPSNET_DTYPE_F32 || x_dtype > UPSNET_DTYPE_PAIR || y_dtype < UPSNET_DTYPE_F32 || y_dtype > UPSNET_DTYPE_PAIR)
    return UPSNET_E_BADARG;
  p.x_bf16 = x_dtype == UPSNET_DTYPE_BF16;
  p.y_bf16 = y_dtype == UPSNET_DTYPE_BF16;
  p.x_pair = x_dtype == UPSNET_DTYPE_PAIR;
  p.y_pair = y_dtype == UPSNET_DTYPE_PAIR;
  p.pair_group = 64 * ((epi_flags >> 8) & 0xfff);
  p.sig_from = ((epi_flags >> 20) & 0x3ff) - 1;
  if (p.sig_from >= 0 && (p.y_pair || p.y_bf16 || p.residual)) return UPSNET_E_UNSUPPORTED;
  // bf16 storage carries precision bf16; hi/lo pairs are the 16-bit storage of precision bf16x3 (the split of x)
  if (p.x_bf16 && p.x3) return UPSNET_E_UNSUPPORTED;
  if ((p.x_pair || p.y_pair) && !p.x3) return UPSNET_E_UNSUPPORTED;
  if (p.y_pair && !p.out_nhwc) return UPSNET_E_BADARG;
  return ups::launch_igemm_tc(p, packed, (cudaStream_t)stream);
}
