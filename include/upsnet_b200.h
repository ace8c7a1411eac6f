/*
 * upsnet_b200.h -- C ABI of libupsnet_b200.so: hand-written sm_90a (H100) CUDA for the UPSNet
 * per-image inference hot path (SURVEY.md section 8).  Plain pointers and sizes only; no
 * torch types.  Every entry point
 *   - takes DEVICE pointers unless the name ends in _host,
 *   - enqueues on `stream` (a cudaStream_t passed as void*) and does not synchronise,
 *   - never allocates (caller-owned outputs and workspaces; sizes from *_workspace_bytes),
 *   - is re-entrant (no global state) and returns 0 on success, a positive cudaError_t
 *     value on a CUDA failure, or a negative UPSNET_E_* code on an argument error.
 * Paths in "replaces:" comments are relative to /root/reference/upsnet/.
 */
#ifndef UPSNET_B200_H_
#define UPSNET_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define UPSNET_E_BADARG (-1)
#define UPSNET_E_UNSUPPORTED (-2)
#define UPSNET_E_WORKSPACE (-3)

#define UPSNET_LAYOUT_NCHW 0
#define UPSNET_LAYOUT_NHWC 1
/* upsnet_roi_align*_forward with UPSNET_DTYPE_PAIR only: out = [R][2][PH*PW*C], the hi plane of the flattened (ph,pw,c)
 * roi feature followed by its lo plane -- i.e. a pair tensor of R 1x1 'images' with PH*PW*C channels (the RCNN fc6 input) */
#define UPSNET_LAYOUT_FLAT_PAIR 2

#define UPSNET_DTYPE_F32 0
#define UPSNET_DTYPE_BF16 1
/* hi/lo bf16 PAIR: an NHWC tensor with 2*C bf16 channels per pixel, [0,C) = bf16(v), [C,2C) = bf16(v - hi) -- the 16-bit
 * storage of precision UPSNET_PREC_BF16X3 (same bytes as fp32, ~16 mantissa bits); v = hi + lo is exact in fp32 */
#define UPSNET_DTYPE_PAIR 2

/* epilogue flags for the convolution entry points */
#define UPSNET_EPI_RELU 1
#define UPSNET_EPI_RES_UP2 2 /* upsnet_igemm_forward only: residual is [N,Ho/2,Wo/2,Cout], read with nearest 2x upsampling */
#define UPSNET_EPI_STEM_PAIR 8 /* upsnet_stem_forward only: y is a hi/lo pair tensor [N,Ho,Wo,2*Cout] (precision bf16x3) */
#define UPSNET_EPI_NO_TMA 4  /* upsnet_igemm_forward only: use the cp.async gather kernel even where the TMA-fed one qualifies */
/* upsnet_group_norm_forward / _backward only, together with UPSNET_EPI_RES_UP2: the half-resolution residual is read
 * with bilinear 2x up-sampling (align_corners = False, as upsnet_upsample2_bilinear_nhwc) instead of nearest */
#define UPSNET_EPI_RES_BILINEAR 16
/* upsnet_igemm_forward, y_dtype PAIR only: store the output channels as [hi G][lo G] per group of G channels instead of
 * [hi Cout][lo Cout] (G % 64 == 0, Cout % G == 0; 0 = Cout).  Lets a 1x1 conv that emulates a 2x2 deconvolution write
 * its four (a,b) sub-pixel groups as four pair pixels (models/rcnn.py:62 mask_deconv1). */
#define UPSNET_EPI_PAIR_GROUP(G) ((((G) / 64) & 0xfff) << 8)
/* upsnet_igemm_forward, fp32 plane-wise (NCHW) or small-Cout outputs only: output channels >= c get a logistic sigmoid
 * 1 / (1 + expf(-v)) after the bias (models/rpn.py:55 cls_prob = sigmoid(cls_score): the RPN head writes the logits and,
 * from duplicated weight rows, their probabilities in one launch). */
#define UPSNET_EPI_SIGMOID_FROM(c) ((((c) + 1) & 0x3ff) << 20)

/* precision of the tensor-core convolution path */
#define UPSNET_PREC_FP32_SIMT 0 /* fp32 FFMA tiles (exact-order-free fp32)            */
#define UPSNET_PREC_BF16X3 1    /* wgmma bf16, 3-term bf16 split (~fp32 result)     */
#define UPSNET_PREC_BF16 2      /* wgmma bf16, single bf16 pass                     */

/* library / build identification: returns 90 for sm_90a, fills `n_sm` if non-NULL */
int upsnet_version(int *n_sm);

/* ---------------------------------------------------------------------------------------
 * ROIAlign forward (sampling grid sr x sr, no half-pixel shift).
 * replaces: operators/src/roi_align_cuda.cpp:39-75 roi_align_forward_cuda
 *           -> operators/src/roi_align_kernel.cu:351 roi_align_forward_gpu_kernel_launcher
 * feat [B,C,H,W] (NCHW) or [B,H,W,C] (NHWC) fp32; rois [R,5] = (batch,x1,y1,x2,y2);
 * out [R,C,PH,PW] (NCHW) or [R,PH,PW,C] (NHWC) -- same layout flag as feat.
 * dtype: UPSNET_DTYPE_F32, or UPSNET_DTYPE_BF16 (NHWC only: bf16 features in, bf16 out, fp32 accumulation), or
 * UPSNET_DTYPE_PAIR (NHWC: hi/lo pair features [B,H,W,2C] in, pair out [R,PH,PW,2C] or UPSNET_LAYOUT_FLAT_PAIR;
 * sampling_ratio > 0, C % 8 == 0).
 */
int upsnet_roi_align_forward(const void *feat, int B, int C, int H, int W, int layout, int dtype,
                             const float *rois, int R, int PH, int PW, int sampling_ratio,
                             float spatial_scale, void *out, void *stream);

/* FPN ROIAlign: level assignment + 4 pyramid levels + un-permute in ONE launch.
 * replaces: operators/modules/fpn_roi_align.py:32-62 FPNRoIAlign.forward (host bucketing,
 *           4 launches, cat, index_select).  feats[l] has spatial size (Hs[l],Ws[l]) and
 *           scale scales[l]; level(roi) = clip(floor(2+log2(sqrt(w*h)/224+1e-6)),0,3).
 * levels_out (optional, may be NULL): int32 [R] chosen level per roi.
 * n_dev (optional, may be NULL; UPSNET_DTYPE_PAIR only): int32 device count -- rois >= *n_dev are neither read nor
 * written (the launch keeps R blocks, so a captured graph does not change shape). */
int upsnet_roi_align_fpn_forward(const void *const feats[4], const int Hs[4], const int Ws[4],
                                 const float scales[4], int B, int C, int layout, int dtype,
                                 const float *rois, int R, int PH, int PW, int sampling_ratio,
                                 void *out, int *levels_out, const int *n_dev, void *stream);

/* ---------------------------------------------------------------------------------------
 * NMS (IoU with the legacy +1 box area, suppress when IoU > thresh).
 * replaces: nms/gpu_nms.hpp:14 _nms  (nms/nms_kernel.cu:40-84 nms_kernel + :97-150 host sweep)
 *
 * Device-resident, segmented: S independent problems in one launch pair.  boxes [total,4]
 * fp32 (x1,y1,x2,y2), already sorted by descending score inside each segment;
 * seg_offsets int32 [S+1] on the DEVICE; max_seg_len = host-known upper bound of a segment
 * length (<= 65536).  keep_out int32 [S, max_seg_len]: positions (relative to the segment
 * start) of kept boxes in ascending order; keep_cnt int32 [S].  Nothing returns to the host.
 */
int upsnet_nms_workspace_bytes(int S, int max_seg_len, size_t *bytes);
int upsnet_nms_segmented(const float *boxes, const int *seg_offsets, int S, int max_seg_len,
                         float thresh, int *keep_out, int *keep_cnt, void *workspace,
                         size_t workspace_bytes, void *stream);
/* Drop-in for the reference's host-pointer entry (same arguments as _nms): boxes_host
 * [n,boxes_dim>=4] sorted by score desc; keep_out/num_out on the host; synchronises. */
int upsnet_nms_host(int *keep_out, int *num_out, const float *boxes_host, int boxes_num,
                    int boxes_dim, float thresh, int device_id);

/* ---------------------------------------------------------------------------------------
 * Deformable convolution v1 / v2 forward, fused (no column buffer in HBM).
 * replaces: operators/functions/deform_conv.py:26-57 DeformConvFunction.forward
 *           (= deform_conv_cuda.deform_im2col, operators/src/deform_conv_cuda.cpp:49-68,
 *              kernel operators/src/deform_conv_kernel.cu:194-242, + torch.mm + bias)
 *           operators/functions/mod_deform_conv.py:25-59 for mask != NULL
 *           (kernel operators/src/mod_deform_conv_kernel.cu:187-249).
 * x [N,Cin,H,W]; offset [N,dg*2*kh*kw,Ho,Wo] (pairs (dh,dw) per tap); mask [N,dg*kh*kw,Ho,Wo]
 * or NULL (already activated: 2*sigmoid); weight [Cout,Cin,kh,kw]; bias [Cout] or NULL;
 * y [N,Cout,Ho,Wo].  All fp32 NCHW contiguous.  groups must be 1 (the reference ignores it).
 */
int upsnet_dcn_forward(const float *x, const float *offset, const float *mask,
                       const float *weight, const float *bias, float *y, int N, int Cin, int H,
                       int W, int Cout, int kh, int kw, int stride_h, int stride_w, int pad_h,
                       int pad_w, int dil_h, int dil_w, int deformable_groups, int epi_flags,
                       int precision, void *stream);

/* Dense convolution forward with fused bias / residual-add / ReLU epilogue (frozen BN is
 * folded into weight+bias by the caller).
 * replaces: the cuDNN conv + BN + ReLU + add chains of models/resnet.py:80-100,
 *           models/fpn.py:78-104, models/rpn.py:52-56, models/rcnn.py:79-87,132-141.
 * x [N,Cin,H,W]; weight [Cout,Cin,kh,kw]; bias/residual may be NULL; residual, y [N,Cout,Ho,Wo]. */
int upsnet_conv2d_forward(const float *x, const float *weight, const float *bias,
                          const float *residual, float *y, int N, int Cin, int H, int W,
                          int Cout, int kh, int kw, int stride_h, int stride_w, int pad_h,
                          int pad_w, int dil_h, int dil_w, int epi_flags, int precision,
                          void *stream);

/* ---------------------------------------------------------------------------------------
 * wgmma implicit-GEMM convolution / deformable convolution (engine entry point).
 * Same arithmetic contract as upsnet_conv2d_forward / upsnet_dcn_forward, but
 *   - x is NHWC [N,H,W,Cin] (Cin % 64 == 0) stored as fp32 or bf16 (x_dtype) -- or, for a tiny Cin <= 8 (the
 *     RGB stem), the fp32 NCHW image itself: K = kh*kw*Cin is flattened and zero-padded to a multiple of 64; y and residual are NHWC or
 *     NCHW (out_layout) stored as fp32 or bf16 (y_dtype); bf16 activations are copied by TMA / cp.async straight
 *     into the tensor-core layout (UPSNET_PREC_BF16); UPSNET_PREC_BF16X3 takes fp32 activations (split in the
 *     gather) or UPSNET_DTYPE_PAIR activations (x [N,H,W,2*Cin], y / residual [N,Ho,Wo,2*Cout]: TMA-fed, three MMAs
 *     per k-slice, fp32 result re-split in the epilogue),
 *   - weights are pre-packed once with upsnet_igemm_pack_weight (bf16 hi/lo planes,
 *     [Cout_pad][kh*kw][Cin]); `packed` must hold upsnet_igemm_packed_weight_bytes bytes,
 *   - offset [N,2*kh*kw,Ho,Wo] / mask [N,kh*kw,Ho,Wo] stay NCHW (reference layout), NULL for a
 *     dense convolution; deformable_groups must be 1,
 *   - precision is UPSNET_PREC_BF16X3 (fp32-grade result) or UPSNET_PREC_BF16,
 *   - n_dev (optional, may be NULL): int32 device count of the images to compute.  On the TMA-fed dense path the tiles
 *     whose first image is >= *n_dev are skipped (a tile holding images on both sides runs in full) and every computed
 *     output is bit-identical to the unbounded launch; the other paths compute all N images.
 * replaces: the same reference call sites as upsnet_conv2d_forward / upsnet_dcn_forward.
 */
int upsnet_igemm_packed_weight_bytes(int Cout, int Cin, int kh, int kw, size_t *bytes);
int upsnet_igemm_pack_weight(const float *weight, int Cout, int Cin, int kh, int kw, void *packed,
                             void *stream);
int upsnet_igemm_forward(const void *x_nhwc, const float *offset, const float *mask,
                         const void *packed, const float *bias, const void *residual, void *y,
                         int N, int H, int W, int Cin, int Cout, int kh, int kw, int stride_h,
                         int stride_w, int pad_h, int pad_w, int dil_h, int dil_w, int out_layout,
                         int x_dtype, int y_dtype, int epi_flags, int precision, const int *n_dev, void *stream);
/* Tuning hook of the TMA-fed dense path of upsnet_igemm_forward (csrc/igemm_tma.cu): output-channel tile of the following
 * launches in this process.  0 (default) = chosen per launch (the widest tile that still gives ~2/3 of the SMs a tile and,
 * for pair activations, a ring of at least three stages); 64 or 128 = that tile wherever Cout rounded up is a multiple of it.
 * A forced tile that does not fit in shared memory is narrowed as the launch's own choice is.  Results are the same for
 * every choice.  UPSNET_E_BADARG for other values. */
int upsnet_tma_set_tile_n(int bn);

/* ---------------------------------------------------------------------------------------
 * Deformable convolution v1 / v2 on hi/lo PAIR activations with the bilinear corners gathered from a shared-memory
 * window (csrc/dcn_win.cu): 3x3, stride 1, deformable_groups 1, Cin % 64 == 0, Cout % 16 == 0, precision
 * UPSNET_PREC_BF16X3.  x [N,H,W,2*Cin] pair NHWC -> y [N,Ho,Wo,2*Cout] pair NHWC; offset / mask as in
 * upsnet_igemm_forward; epi_flags: UPSNET_EPI_RELU.  Same arithmetic contract as upsnet_igemm_forward with an offset
 * (samples outside the staged window are gathered from global memory: the result does not depend on the window size).
 * `packed` comes from upsnet_dcn_pack_weight (K order: 16-channel sub-chunk, tap, channel) and holds
 * upsnet_dcn_packed_weight_bytes bytes.  All three return UPSNET_E_UNSUPPORTED for other layer shapes: callers then use
 * upsnet_igemm_forward.
 * replaces: operators/functions/deform_conv.py:26-57 (deformable_im2col + torch.mm),
 *           operators/src/deform_conv_kernel.cu:89-118,194-242, mod_deform_conv_kernel.cu (v2 mask). */
int upsnet_dcn_packed_weight_bytes(int Cout, int Cin, int kh, int kw, size_t *bytes);
int upsnet_dcn_pack_weight(const float *weight, int Cout, int Cin, int kh, int kw, void *packed, void *stream);
int upsnet_dcn_pair_forward(const void *x_pair, const float *offset, const float *mask, const void *packed,
                            const float *bias, void *y_pair, int N, int H, int W, int Cin, int Cout, int kh, int kw,
                            int pad_h, int pad_w, int dil_h, int dil_w, int epi_flags, void *stream);
/* Tuning hook of upsnet_dcn_pair_forward: output-channel tile of the following launches in this process.  0 (default) =
 * chosen per launch (128 when Cout is a multiple of 128 and the layer has at least a quarter as many 16x8-pixel tiles as
 * the GPU has SMs, else 32); 32 or 128 = that tile wherever it applies (128 needs Cout rounded up to 64 to be a multiple of 128).  Results are
 * the same for every choice.  UPSNET_E_BADARG for other values. */
int upsnet_dcn_set_tile_n(int bn);

/* ---------------------------------------------------------------------------------------
 * Parameter-free panoptic head, fused: MaskRemoval + SegTerm + void/concat/argmax.
 * replaces: models/resnet_upsnet.py:223-240 with operators/modules/mask_removal.py:29-93,
 *           operators/modules/unary_logits.py:78-105.  Never materialises the [1,k,H,W] planes.
 * fcn [S,H,W] fp32 (fcn_output of one image); boxes [n,4] (mask_rois[:,1:]); cls_prob [n];
 * mask_logit [n,28,28] (logit of the predicted class); cls_idx int64 [n] (1-based thing class,
 * <= num_thing); num_stuff = S - num_thing.
 * n is the (maximum) instance count known to the host; n_dev (optional, may be NULL) is a DEVICE int32 with
 * the actual count <= n, so the call can be enqueued without knowing it (static-shape engine / CUDA graphs).
 * keep_out int64 [max(n,1)] original indices of kept instances in score order, k_out int32[1];
 * labels int64 [H,W] (255 = void); sem_labels int64 [H,W] or NULL (argmax_c fcn).
 * Workspace: upsnet_panoptic_workspace_bytes is the preferred size (the 1-bit mask windows of all n instances resident,
 * capped at 64 MB); any size >= upsnet_panoptic_workspace_min_bytes is accepted -- the windows are then built and
 * consumed in rounds of consecutive score ranks (at most 64), with identical results.
 */
int upsnet_panoptic_workspace_bytes(int n, int H, int W, int num_thing, size_t *bytes);
int upsnet_panoptic_workspace_min_bytes(int n, int H, int W, int num_thing, size_t *bytes);
int upsnet_panoptic_head(const float *fcn, int S, int H, int W, const float *boxes,
                         const float *cls_prob, const float *mask_logit, const int64_t *cls_idx,
                         int n, const int *n_dev, int num_stuff, double fraction_threshold, int64_t *keep_out,
                         int *k_out, int64_t *labels, int64_t *sem_labels, void *workspace,
                         size_t workspace_bytes, void *stream);
/* Same head on the QUARTER-resolution score map: score [S,Hs,Ws] (models/fcn.py:94-101 `score` before the final
 * nn.Upsample(scale_factor=4, mode='bilinear')), labels / sem_labels [4*Hs,4*Ws].  The up-sampling is evaluated inside the
 * fusion kernel with the arithmetic of upsnet_upsample_bilinear_nchw (factor 4), so the results are bit-identical to
 * upsnet_panoptic_head on the materialised [S,4*Hs,4*Ws] logits, which are neither written nor read (159 MB each way at
 * 19 x 1024 x 2048).  Workspace sizes: upsnet_panoptic_workspace_bytes(n, 4*Hs, 4*Ws, num_thing). */
int upsnet_panoptic_head_up4(const float *score, int S, int Hs, int Ws, const float *boxes,
                             const float *cls_prob, const float *mask_logit, const int64_t *cls_idx,
                             int n, const int *n_dev, int num_stuff, double fraction_threshold, int64_t *keep_out,
                             int *k_out, int64_t *labels, int64_t *sem_labels, void *workspace,
                             size_t workspace_bytes, void *stream);

/* MaskRemoval alone (API parity with operators/modules/mask_removal.py:29-93): score-ordered overlap
 * pruning; keep_out / k_out as above; mask_energy (optional, may be NULL) float [n,H,W]: planes 0..k-1
 * receive the pasted, resized logits of the kept instances (zeros elsewhere), as the reference returns
 * them.  Workspace size: upsnet_panoptic_workspace_bytes. */
int upsnet_mask_removal(const float *boxes, const float *cls_prob, const float *mask_logit,
                        const int64_t *cls_idx, int n, const int *n_dev, int H, int W, int num_thing,
                        double fraction_threshold, int64_t *keep_out, int *k_out, float *mask_energy,
                        void *workspace, size_t workspace_bytes, void *stream);

/* RGB stem on the TMA kernel: k x k (kw <= 8) / stride 2 / pad `pad` convolution of a tiny-Cin (<= 8) fp32 NCHW
 * image, bf16 NHWC output [N,Ho,Wo,Cout] (Cout % 64 == 0) -- or, with UPSNET_EPI_STEM_PAIR, the hi/lo pair tensor
 * [N,Ho,Wo,2*Cout] computed with the three-pass split from hi/lo copies of the image -- fused bias + ReLU (UPSNET_EPI_RELU).
 * replaces: models/resnet.py:155-162 conv1 + bn1 (folded) + relu.
 * The call first packs the image to a zero-padded bf16 NHWC8 copy in `workspace` (upsnet_stem_workspace_bytes),
 * then runs the wgmma kernel whose A tiles are boxes of a 5-D tensor map over that copy; weights are packed
 * once with upsnet_stem_pack_weight ([Cout][kh][8][8] bf16, upsnet_stem_packed_weight_bytes).
 * Returns UPSNET_E_UNSUPPORTED if the driver rejects the tensor map (callers fall back to upsnet_igemm_forward). */
int upsnet_stem_workspace_bytes(int N, int H, int W, int kh, int kw, int pad, size_t *bytes);
int upsnet_stem_packed_weight_bytes(int Cout, int kh, size_t *bytes);
int upsnet_stem_pack_weight(const float *weight, int Cout, int Cin, int kh, int kw, void *packed,
                            void *stream);
int upsnet_stem_forward(const float *x, const void *packed_w, const float *bias, void *y, int N, int Cin,
                        int H, int W, int Cout, int kh, int kw, int pad, int epi_flags, void *workspace,
                        size_t workspace_bytes, void *stream);

/* Max-pooling on NHWC activations (bf16, hi/lo pair or fp32 storage; C % 8 == 0 resp. C % 4 == 0), floor output size.
 * UPSNET_DTYPE_PAIR: x [N,H,W,2C] -> y [N,Ho,Wo,2C], the window element with the largest hi + lo is copied.
 * replaces: models/resnet.py:163 nn.MaxPool2d(kernel_size=3, stride=2, padding=1) of the stem.
 * x [N,H,W,C] -> y [N,Ho,Wo,C], Ho = (H + 2*pad - k)/stride + 1; padding never wins the max. */
int upsnet_maxpool2d_nhwc(const void *x, void *y, int N, int H, int W, int C, int k, int stride,
                          int pad, int dtype, void *stream);

/* Bilinear up-sampling by an integer factor, NCHW fp32 planes, align_corners = False.
 * replaces: models/fcn.py:88-101 nn.Upsample(scale_factor=4, mode='bilinear') of the semantic logits
 *           (source index (dst + 0.5)/factor - 0.5 clamped at 0, as ATen's upsample_bilinear2d).
 * x [planes,H,W] -> y [planes,H*factor,W*factor]; (W*factor) % 4 == 0. */
int upsnet_upsample_bilinear_nchw(const float *x, float *y, int planes, int H, int W, int factor,
                                  void *stream);

/* Semantic-head score assembly: out = s2 + up2(s3) + up4(s4) + up8(s5), bilinear, align_corners = False.
 * replaces: models/fcn.py:94-101 (three F.interpolate of 128-channel maps + cat + score conv; the engine scores every level
 *           at its own resolution first -- the 1x1 conv and the up-sampling commute -- and sums the 19-plane maps here).
 * s2 [planes,H,W], s3 [planes,H/2,W/2], s4 [planes,H/4,W/4], s5 [planes,H/8,W/8] fp32; H % 8 == W % 8 == 0. */
int upsnet_fcn_score_fuse(const float *s2, const float *s3, const float *s4, const float *s5, float *out,
                          int planes, int H, int W, void *stream);

/* The adjoint of upsnet_fcn_score_fuse (the semantic head's backward through the level sum):
 * ds3 = up2^T(dscore), ds4 = up4^T(dscore), ds5 = up8^T(dscore) with the forward's bilinear weights (align_corners =
 * False, clamped at 0, the last row / column repeated); d s2 is dscore itself, so nothing is written for it.
 * replaces: autograd of the three F.interpolate of models/fcn.py:94-96 behind the score conv.
 * dscore [planes,H,W] -> ds3 [planes,H/2,W/2], ds4 [planes,H/4,W/4], ds5 [planes,H/8,W/8] fp32, every element written.
 * One launch.  A gather in a fixed order, no atomics: the same inputs give the same bytes; capturable.
 * H % 8 == W % 8 == 0 and planes <= 65535, else UPSNET_E_UNSUPPORTED. */
int upsnet_fcn_score_fuse_backward(const float *dscore, float *ds3, float *ds4, float *ds5, int planes, int H,
                                   int W, void *stream);

/* FPN top-down bilinear 2x up-sampling on NHWC activations (csrc/upsample2.cu), align_corners = False: the rule of
 * upsnet_upsample_bilinear_nchw with factor 2 (source index (dst + 0.5)/2 - 0.5 clamped at 0, the last row / column
 * repeated; any h, w, odd ones included).
 * replaces: models/fpn.py:27-35 fpn_upsample with network.fpn_upsample_method = 'bilinear', applied at :88-93.
 * x [N,h,w,C] -> y [N,2h,2w,C] in dtype (F32, BF16, or PAIR: [N,h,w,2C] -> [N,2h,2w,2C]); interpolated in fp32 (a
 * pair's value is hi + lo) and rounded once to dtype.  C % 8 == 0 and 16-byte aligned x, y, else UPSNET_E_UNSUPPORTED.
 *
 * upsnet_upsample2_bilinear_nhwc_adjoint: dx = up2^T(dy), fp32 NHWC dy [N,2h,2w,C] -> dx [N,h,w,C], every element
 * written.  A gather (each coarse pixel sums its 4x4 fine footprint with the forward's weights, along x then y, in a
 * fixed order), no atomics: the same input gives the same bytes; capturable.  C % 4 == 0 and 16-byte aligned dy, dx,
 * else UPSNET_E_UNSUPPORTED.
 * replaces: autograd of that F.interpolate. */
int upsnet_upsample2_bilinear_nhwc(const void *x, void *y, int N, int h, int w, int C, int dtype, void *stream);
int upsnet_upsample2_bilinear_nhwc_adjoint(const float *dy, float *dx, int N, int h, int w, int C, void *stream);

/* ---------------------------------------------------------------------------------------
 * Detection glue, fused (device-resident; nothing returns to the host).
 *
 * upsnet_rpn_decode: anchors + deltas -> clipped proposal boxes for the pre-NMS top-k of every pyramid level.
 * replaces: operators/functions/pyramid_proposal.py:83-131 (shifted anchors, bbox_transform, clip_boxes;
 *           bbox/bbox_transform.py:290-330,45-60) for the selected indices.
 * deltas[l] fp32 [4A,h_l,w_l] (RPN head output, channel a*4+c); top_idx[l] int64 [k_l] flat (y,x,a) indices
 * (device); k/hs/ws/strides host arrays [L]; base_anchors float64 [L,A,4] on the device (generate_anchors);
 * im_info fp32 [3] on the device: the reference's (h, w, scale) row; boxes are clipped to [0, w-1] x [0, h-1].  It is
 * read when the kernel runs, so a captured graph takes a new image size by rewriting the row before each replay.
 * boxes_out fp32 [sum k_l, 4] in level order. */
int upsnet_rpn_decode(const float *const *deltas, const long long *const *top_idx, const int *k,
                      const int *hs, const int *ws, const int *strides, const double *base_anchors,
                      int L, int A, const float *im_info, float *boxes_out, void *stream);

/* upsnet_rpn_topk: the pre_nms_top_n best anchors of every pyramid level, sorted by descending score, one call.
 * replaces: operators/functions/pyramid_proposal.py:104-118 (per-level argsort(-scores)[:pre_nms_top_n]).
 * probs[l] fp32 [A,h_l,w_l] (device); k_l = min(pre_nms_top_n, A*h_l*w_l) <= 2048; out_scores fp32 / out_idx int64
 * [sum k_l]: level after level, flat (y,x,a) indices as the reference's transposed score vector uses; equal
 * scores are ordered by ascending index.  Workspace: upsnet_rpn_topk_workspace_bytes(L). */
int upsnet_rpn_topk_workspace_bytes(int L, size_t *bytes);
int upsnet_rpn_topk(const float *const *probs, const int *hs, const int *ws, int L, int A,
                    int pre_nms_top_n, float *out_scores, long long *out_idx, void *workspace,
                    size_t workspace_bytes, void *stream);

/* upsnet_rpn_collect: per level the first min(keep_cnt, post_nms_top_n) NMS survivors, then the post_nms_top_n
 * best of their union by score (descending), as fixed-size outputs.
 * replaces: operators/functions/pyramid_proposal.py:196-222 + modules/pyramid_proposal.py:61-67.
 * keep/keep_cnt/seg_offsets from upsnet_nms_segmented over (boxes, scores) [total]; rois fp32 [post,5] =
 * (0,x1,y1,x2,y2), rows past the live count are zero; out_scores [post]; valid uint8 [post]. */
int upsnet_rpn_collect(const int *keep, const int *keep_cnt, const int *seg_offsets, const float *boxes,
                       const float *scores, int S, int max_seg_len, int post_nms_top_n, float *rois,
                       float *out_scores, unsigned char *valid, void *stream);

/* upsnet_maskroi_prepare: candidate selection (prob > score_thresh, roi valid), ordering (class segment
 * ascending -- one segment when class_agnostic --, score descending, roi-major index ascending) and box decode
 * (weights, clip) in one launch.  replaces: operators/modules/mask_roi.py:36-95 up to the per-class NMS.
 * rois [R,5]; roi_valid uint8 [R]; bbox_delta [R,4C]; cls_prob [R,C]; R*(C-1) <= 8192; im_info fp32 [3] on the
 * device, (h, w, scale), read when the kernel runs (as in upsnet_rpn_decode): boxes are clipped to [0, w-1] x [0, h-1].
 * sc_out/cls_out/bx_out [R*(C-1)] (/[.,4]): candidates first, in NMS input order (others: score -1);
 * offs_out int32 [nseg+1]: segment offsets for upsnet_nms_segmented. */
int upsnet_maskroi_prepare(const float *rois, const unsigned char *roi_valid, const float *bbox_delta,
                           const float *cls_prob, int R, int C, int class_agnostic, float score_thresh,
                           const float weights[4], const float *im_info, float *sc_out, int *cls_out,
                           float *bx_out, int *offs_out, void *stream);

/* upsnet_maskroi_finish: NMS survivors (class-major) -> keep scores >= the top_n-th largest -> `cap` output
 * slots (score, (0,x1,y1,x2,y2), class) + device count; no survivor -> one dummy detection (score 1, zero box,
 * class 0).  replaces: operators/modules/mask_roi.py:96-139.  keep/keep_cnt/seg_offsets as produced by
 * upsnet_nms_segmented on bx; nseg <= 128.  n_out int32 [2]: [0] = number of detections, [1] = truncation flags (the
 * reference keeps every survivor and every box tied at the top-n threshold): bit 0 = more NMS survivors than the 4096
 * candidate slots, bit 1 = more boxes at / above the threshold than `cap` output slots. */
int upsnet_maskroi_finish(const int *keep, const int *keep_cnt, const int *seg_offsets, const float *sc,
                          const int *cls, const float *bx, int nseg, int max_seg_len, int top_n, int cap,
                          float *out_sc, float *out_bx, long long *out_cls, int *n_out, void *stream);

/* upsnet_mask_rows: the rows the mask branch has to compute for one image, from the two MaskROI outputs (b1 [cap1,5], device
 * count n1: detections; b2 [cap2,5], device count n2: panoptic candidates).  A row's logits depend on its box alone, so a
 * candidate whose box (all five floats, compared bit for bit) equals a detection's box takes that detection's row.
 * rows [cap1+cap2,5]: the n1 detections in order, then the candidates that match no detection in order, then zeros;
 * u int32 device scalar: the number of rows written before the zeros; pan_row int32 [cap2]: the row of candidate j's logits
 * (0 for j >= n2).  Counts are clamped to [0, cap].  One CTA, deterministic, no host read (graph-capturable).
 * replaces: models/resnet_upsnet.py:203-222 running the mask branch once on the detections and once on the candidates. */
int upsnet_mask_rows(const float *b1, const int *n1, int cap1, const float *b2, const int *n2, int cap2, float *rows,
                     int *u, int *pan_row, void *stream);

/* ---------------------------------------------------------------------------------------
 * Callers either side of the per-image forward (SURVEY section 8f), device resident.
 *
 * upsnet_unified_pan_result: the 2-channel panoptic result the PQ evaluation consumes.
 * replaces: dataset/base_dataset.py:332-371 get_unified_pan_result (numpy on the host: np.unique per segment).
 * seg int64 [H,W] (semantic argmax, 'fcn_outputs'), pan int64 [H,W] ('panoptic_outputs': 0..id_last_stuff stuff,
 * id_last_stuff + 1 + j = j-th kept instance, 255 void; id_last_stuff = num_seg_classes - num_classes), cls_inds int64
 * [k] ('panoptic_cls_inds', 1-based thing class of kept instance j); k_dev optional DEVICE count <= k.
 * pan_2ch uint8 [H,W,3]: channel 0 = semantic class (255 void), 1 = instance number (rank among the instance ids present,
 * from 1; 0 = stuff), 2 = 0.  A segment takes its semantic majority class when that is a stuff class holding >= half of
 * it; stuff classes smaller than stuff_area_limit pixels become void.  err_out (optional DEVICE int): bit 0 = label out of
 * range, bit 1 = an instance id without an entry in cls_inds (the reference raises IndexError).
 */
int upsnet_unified_pan_workspace_bytes(int num_seg_classes, size_t *bytes);
int upsnet_unified_pan_result(const long long *seg, const long long *pan, const long long *cls_inds, int k,
                              const int *k_dev, int H, int W, int num_seg_classes, int num_classes,
                              int stuff_area_limit, unsigned char *pan_2ch, int *err_out, void *workspace,
                              size_t workspace_bytes, void *stream);

/* upsnet_prep_image: raw uint8 HWC (BGR) image -> the network input blob.
 * replaces: dataset/base_dataset.py:143-174 prep_im_for_blob (mean subtraction, cv2.resize INTER_LINEAR) and :898-923
 *           im_list_to_blob (zero padding to a multiple of the FPN stride, HWC -> CHW), plus the 4x larger fp32 H2D copy.
 * image_hwc uint8 [h,w,3] on the DEVICE; scale = the fx = fy factor handed to cv2.resize (the source step is 1/scale,
 * as OpenCV does when factors are given); (out_h,out_w) = the resized size (cvRound(h*scale), cvRound(w*scale));
 * (pad_h,pad_w) >= it; blob fp32 [3,pad_h,pad_w]: resized (image - pixel_means), zeros in the padding.  The means are
 * float64 like config.network.pixel_means: numpy subtracts in double and stores float32 (base_dataset.py:154).
 * flip != 0: the image is mirrored first, as get_image_blob does for a flipped roidb entry (base_dataset.py:128-129,
 * im[:, ::-1, :]): source column x is read as w - 1 - x before the mean subtraction and the bilinear taps, so the blob
 * equals, bit for bit, the one of a host-flipped copy with flip = 0.
 */
int upsnet_prep_image(const unsigned char *image_hwc, int h, int w, double scale, int out_h, int out_w, int pad_h,
                      int pad_w, const double pixel_means[3], float *blob, int flip, void *stream);

/* upsnet_label_restore: a network-resolution label map back to the original image size.
 * replaces: upsnet_end2end_test.py:259-266 -- crop [:h,:w], astype(uint8) (values wrap mod 256), cv2.resize(fx = fy,
 *           INTER_NEAREST) on the host.
 * src0 / src1 int64 [Hp,Wp] (src1 / dst1 may be NULL: both maps of an image in one launch); (h,w) <= (Hp,Wp) the crop;
 * fx the resize factor (the caller passes cv2's double); out_h = rint(h*fx), out_w = rint(w*fx) (half to even, cvRound).
 * dst int64 [out_h,out_w] = (uint8) src[min(floor(y/fx),h-1)][min(floor(x/fx),w-1)] with 1/fx taken in double. */
int upsnet_label_restore(const long long *src0, const long long *src1, int Hp, int Wp, int h, int w, double fx,
                         int out_h, int out_w, long long *dst0, long long *dst1, void *stream);

/* ---------------------------------------------------------------------------------------
 * Panoptic quality statistics of one image on the device (SURVEY section 8 row f4, evaluation half).
 * replaces: dataset/base_dataset.py:462-511 _converter_2ch_single_core + :513-608 _pq_compute_single_core (numpy on the
 *           host: np.unique over the 2-channel map, one full-image mask per segment, np.unique over a uint64 pair map).
 * pan_2ch uint8 [H,W,3] (class, instance, -) as upsnet_unified_pan_result writes it; class 255 = void.  A prediction
 *   segment is (class, instance) for a thing class and the class alone for a stuff class (stuff instances merge).
 * gt_rgb uint8 [H,W,3], id = R + 256 G + 65536 B; id 0 = VOID.
 * gt_table int64 [5][num_gt] (structure of arrays): id, category_id, iscrowd, area, order.  Rows sorted by strictly
 *   ascending id in [1, 2^24); `order` = the row's position in the ground truth's segment list after duplicate ids are
 *   merged the way a Python dict does (the later entry wins, the first position is kept); category_id in [0,255).
 * cat_flags uint8 [256]: bit 0 = category known, bit 1 = isthing.
 * acc_counts int64 [3][256] (tp, fp, fn per category id) and acc_iou fp64 [256] are ADDED to; the per-match IoUs are
 *   summed in ascending (gt id, prediction segment) order, so repeated runs give bit-identical sums.
 * err (DEVICE int, sticky: bits are OR-ed in, never cleared): UPSNET_PQ_E_* below.  The call never synchronises.
 * Workspace: upsnet_pq_workspace_bytes. */
#define UPSNET_PQ_MAX_GT 4096        /* ground-truth segments per image */
#define UPSNET_PQ_MAX_PAIRS 65536    /* distinct (ground-truth segment, prediction segment) pairs per image */
#define UPSNET_PQ_MAX_PRED 2048      /* prediction segments per image */
#define UPSNET_PQ_E_PRED_CATEGORY 1  /* a prediction class that is neither 255 nor a known category */
#define UPSNET_PQ_E_GT_COUNT 2       /* num_gt > UPSNET_PQ_MAX_GT */
#define UPSNET_PQ_E_PAIRS 4          /* more than UPSNET_PQ_MAX_PAIRS distinct pairs */
#define UPSNET_PQ_E_GT_TABLE 8       /* ids not strictly ascending in [1,2^24), or a category id outside [0,255) */
#define UPSNET_PQ_E_PRED_COUNT 16    /* more than UPSNET_PQ_MAX_PRED prediction segments */
#define UPSNET_PQ_E_MATCHES 32       /* more than UPSNET_PQ_MAX_GT matches (only when table areas undercount pixels) */
int upsnet_pq_workspace_bytes(size_t *bytes);
int upsnet_pq_update(const unsigned char *pan_2ch, const unsigned char *gt_rgb, int H, int W, const long long *gt_table,
                     int num_gt, const unsigned char *cat_flags, long long *acc_counts, double *acc_iou, int *err,
                     void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------
 * Semantic-segmentation confusion matrix of one image on the device (SURVEY section 8 row f4, evaluation half).
 * replaces: dataset/cityscapes.py:445-514 / coco.py:225-293 evaluate_ssegs + write_segmentation_result and
 *           base_dataset.py:806-824 get_confusion_matrix (a PNG per prediction, PIL NEAREST resize to the ground-truth
 *           size, np.bincount on the host).
 * pred [rows][pred_pitch] elements of pred_bytes = 1 (uint8) or 8 (int64); each value is wrapped to uint8 (np.uint8).
 * row_src int32 [H], col_src int32 [W]: the prediction element of gt pixel (y, x) is pred[row_src[y] * pred_pitch +
 *   col_src[x]]; every resize / restore rule lives in these tables, which the caller builds (indices are not checked).
 * gt uint8 [H,W]; pixels with gt == 255 are ignored.  A pixel counts in bin gt * C + pred only if that is < C*C (so gt
 *   rows >= C drop and predictions >= C alias into later rows, as in the reference).
 * acc int64 [C*C] (row = gt, column = prediction) is ADDED to with integer atomics: the result is order independent.
 * 1 <= num_classes <= UPSNET_SSEG_MAX_CLASSES (a C*C uint32 histogram per block in shared memory).  No workspace; the
 * call never synchronises. */
#define UPSNET_SSEG_MAX_CLASSES 224
int upsnet_sseg_update(const void *pred, int pred_bytes, int pred_pitch, const int *row_src, const int *col_src,
                       const unsigned char *gt, int H, int W, int num_classes, long long *acc, void *stream);

/* ---------------------------------------------------------------------------------------
 * COCO box and mask AP on the device (SURVEY section 8 row f4, evaluation half).
 * replaces: dataset/base_dataset.py:181-204 evaluate_boxes / coco.py:194-222 evaluate_masks -- a results JSON written,
 *           reloaded with COCO.loadRes and scored by pycocotools' COCOeval.evaluate() / accumulate() on the host.
 * Semantics: COCOeval with its default Params (iouThrs linspace(.5,.95,10), recThrs linspace(0,1,101), maxDets 1/10/100,
 *   area ranges all / small / medium / large, useCats), none of which is a parameter here.
 *
 * upsnet_cocoeval_image: evaluate() of one image.  Detections: boxes fp32 [n][4] xyxy, scores fp32 [n], cls_inds int64 [n]
 *   (class j in [1, num_categories]; K index class_to_k[j], class_to_k int32 [num_categories + 1] on the device); only
 *   the first min(n, *n_dev) count when n_dev (device int) is given.  segm != 0: masks are counts uint32 [n][cap] /
 *   run_len int32 [n] exactly as upsnet_im_post_rle leaves them, of an H x W image.
 *   gt_table fp64 [9][num_gt] (structure of arrays): K index, iscrowd, area (the annotation's field), x, y, w, h, and for
 *   segm the RLE's h, w.  segm: gt_counts uint32 (uncompressed run lengths, all ground truths back to back), gt_offsets
 *   int64 [num_gt + 1].  The workspace (segm only) is upsnet_cocoeval_workspace_bytes(n, cap, gt_offsets[num_gt]).
 *   Writes one record per kept detection (the first 100 of its category by descending score, ties in input order) at
 *   records[atomicAdd(n_records, ...)]; bit a * 10 + t of matched / ignored is evaluateImg's dtMatches != 0 / dtIgnore for
 *   IoU threshold t and area range a.  npig int64 [num_categories][4] is ADDED to (non-ignored ground truths).
 *   Limits: UPSNET_COCOEVAL_MAX_DET detections, UPSNET_COCOEVAL_MAX_GT ground truths per image, UPSNET_COCOEVAL_MAX_GT_CAT
 *   per (image, category), record_cap records.  err (DEVICE int, sticky) gets UPSNET_COCOEVAL_E_*; nothing is truncated
 *   silently.  The call never synchronises.
 * upsnet_cocoeval_accumulate: accumulate() over records [n_records].  image_rank int32 [image slot] = rank of the slot's
 *   image id among all image ids (< UPSNET_COCOEVAL_MAX_IMAGES).  Writes precision / scores fp64 [10][101][K][4][3] and
 *   recall fp64 [10][K][4][3], numpy's C order.  Workspace: upsnet_cocoeval_accumulate_workspace_bytes(n_records). */
#define UPSNET_COCOEVAL_MAX_DET 2048
#define UPSNET_COCOEVAL_MAX_GT 1024
#define UPSNET_COCOEVAL_MAX_GT_CAT 192
#define UPSNET_COCOEVAL_MAX_CATEGORIES 256
#define UPSNET_COCOEVAL_MAX_IMAGES (1 << 17)
#define UPSNET_COCOEVAL_E_DET_COUNT 1   /* more than UPSNET_COCOEVAL_MAX_DET detections */
#define UPSNET_COCOEVAL_E_GT_COUNT 2    /* num_gt > UPSNET_COCOEVAL_MAX_GT */
#define UPSNET_COCOEVAL_E_GT_CAT 4      /* more than UPSNET_COCOEVAL_MAX_GT_CAT ground truths of one category */
#define UPSNET_COCOEVAL_E_CLASS 8       /* a detection class outside [1, num_categories] */
#define UPSNET_COCOEVAL_E_RECORDS 16    /* more than record_cap records */
#define UPSNET_COCOEVAL_E_RLE_SIZE 32   /* an RLE that does not cover the H x W image, or run_len > cap */
typedef struct {
  float score;
  int category;                         /* K index */
  int image;                            /* image slot */
  int rank;                             /* rank in (image, category), < 100 */
  unsigned long long matched, ignored;  /* bit a * 10 + t */
} upsnet_coco_record;
int upsnet_cocoeval_workspace_bytes(int n, int cap, long long gt_counts_total, size_t *bytes);
int upsnet_cocoeval_image(int segm, const float *boxes, const float *scores, const int64_t *cls_inds, int n,
                          const int *n_dev, const uint32_t *counts, int cap, const int *run_len, int H, int W,
                          const double *gt_table, int num_gt, const uint32_t *gt_counts, const int64_t *gt_offsets,
                          int num_categories, const int *class_to_k, int image_slot, upsnet_coco_record *records,
                          int record_cap, int *n_records, long long *npig, int *err, void *workspace,
                          size_t workspace_bytes, void *stream);
/* upsnet_gt_rle: the ground truths of one image as upsnet_cocoeval_image reads them, COCO.annToRLE on the device
 * (maskUtils.merge(maskUtils.frPyObjects(segm, h, w)) for a list segmentation).
 *   Annotation g (of num_anns, in annotation order) is the union of polygons [ann_poly[g], ann_poly[g+1]) (ann_poly int32
 *   [num_anns + 1]); polygon q has the fp64 vertices verts[poly_vert[q] .. poly_vert[q+1]) (poly_vert int32 [P + 1],
 *   verts (x, y) pairs, |coordinate| < 4e8).  Each polygon is rasterised as maskApi.c rleFrPoly does at h x w (k =
 *   its vertex count, 0 and 1 included), and the polygons are united as rleMerge(..., intersect = 0).  A box-list
 *   segmentation is passed as rleFrBbox's polygons [xs, ys, xs, ye, xe, ye, xe, ys].  An annotation without polygons
 *   takes src_counts[src_offsets[g] .. src_offsets[g+1]) (uint32, src_offsets int64 [num_anns + 1]) unchanged: the
 *   uncompressed run lengths of an RLE segmentation, staged from the host.
 *   Writes gt_counts uint32 (all annotations back to back, the canonical runs: column-major, zeros first, the first run
 *   possibly 0, every later one > 0, summing to h * w) and gt_offsets int64 [num_anns + 1].  capacity: the gt_counts
 *   elements available, at least the total run count; for an annotation of polygons, 1 + the sum over its edges of
 *   min(w, (|X1 - X0| + 1) / 5 + 1) with X = (int)(5 x + .5) bounds its runs.  Over capacity: err (DEVICE int,
 *   sticky) gets UPSNET_GT_RLE_E_CAPACITY, every offset is 0 and no run is written.  Offsets come from a device scan;
 *   the call never synchronises.  Deterministic: the same input gives the same bytes.
 *   Limits: h, w >= 1 and h * w < 2^31, num_anns <= 65535 (else UPSNET_E_UNSUPPORTED).
 *   Workspace: upsnet_gt_rle_workspace_bytes(num_anns, h, w). */
#define UPSNET_GT_RLE_E_CAPACITY 64   /* more runs than capacity (the bit is free in the UPSNET_COCOEVAL_E_* flag) */
int upsnet_gt_rle_workspace_bytes(int num_anns, int h, int w, size_t *bytes);
int upsnet_gt_rle(int h, int w, int num_anns, const int *ann_poly, const int *poly_vert, const double *verts,
                  const int64_t *src_offsets, const uint32_t *src_counts, uint32_t *gt_counts, long long capacity,
                  int64_t *gt_offsets, int *err, void *workspace, size_t workspace_bytes, void *stream);
int upsnet_cocoeval_accumulate_workspace_bytes(int n_records, size_t *bytes);
int upsnet_cocoeval_accumulate(const upsnet_coco_record *records, int n_records, const int *image_rank,
                               const long long *npig, int num_categories, double *precision, double *recall,
                               double *scores, void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------
 * upsnet_combined_pan_result: the combined panoptic result (instance output merged heuristically with the semantic head).
 * replaces: dataset/base_dataset.py:373-449 get_combined_pan_result + _merge_pred_single_core (every detection decoded
 *           to a full [H,W] image with pycocotools and three full-image boolean passes per detection, on the host).
 * sem [H,W] of sem_elem_size = 1 (uint8) or 8 (int64, each value wrapped to uint8), the restored semantic map;
 *   H * W <= 2^24 (the float32 pixel counts of the reference are exact up to there).
 * Detections: scores fp32 [n], cls_inds int64 [n]; only the first min(n, *n_dev) count when n_dev (device int) is given,
 *   and of those only classes in [1, num_classes) (the ones im_post keeps).  Masks: counts uint32 [n][cap] / run_len
 *   int32 [n] exactly as upsnet_im_post_rle leaves them, of an H x W image.
 * Order: descending score; among equal scores the detection later in the class-ascending concatenation of im_post's
 *   per-class lists first, i.e. (score desc, class desc, index desc) -- np.argsort(score, kind='stable')[::-1].
 * A detection is skipped when score < score_threshold, when its mask is empty, or when (float32) remain / area <
 *   fraction_threshold, remain = its pixels not claimed by an earlier kept detection.  A kept detection of class c gets
 *   instance number (++count[c]) mod 256 and claims its free pixels; number 0 (the 256th, ...) claims nothing.
 * pan_2ch uint8 [H,W,3]: channel 0 = the semantic class, 255 where a class <= id_last_stuff (= num_seg_classes -
 *   num_classes) has fewer than stuff_area_limit pixels or where a class > id_last_stuff has no instance, and
 *   (c + id_last_stuff) mod 256 on the pixels of an instance of class c; channel 1 = the instance number; channel 2 = 0.
 * err (DEVICE int, sticky): UPSNET_COMBINED_E_* below; a detection whose runs are unusable is skipped, more than
 *   UPSNET_COMBINED_MAX_DET detections skips them all.  The call never synchronises.
 * Workspace: upsnet_combined_pan_workspace_bytes(n, H, W) (a histogram, an H*W-bit occupancy bitmap and a 2-byte owner
 * per pixel). */
#define UPSNET_COMBINED_MAX_DET 2048
#define UPSNET_COMBINED_E_RUN_LEN 1     /* run_len > cap (upsnet_im_post_rle overflowed its buffer) or < 0 */
#define UPSNET_COMBINED_E_RLE_SIZE 2    /* runs that do not sum to H * W */
#define UPSNET_COMBINED_E_DET_COUNT 4   /* more than UPSNET_COMBINED_MAX_DET detections */
int upsnet_combined_pan_workspace_bytes(int n, int H, int W, size_t *bytes);
int upsnet_combined_pan_result(const void *sem, int sem_elem_size, int H, int W, const float *scores,
                               const int64_t *cls_inds, int n, const int *n_dev, const uint32_t *counts, int cap,
                               const int *run_len, int num_seg_classes, int num_classes, float score_threshold,
                               float fraction_threshold, int stuff_area_limit, unsigned char *pan_2ch, int *err,
                               void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------
 * Instance-mask post-processing of the test loop on the device (SURVEY section 8 row f4).
 * replaces: upsnet_end2end_test.py:95-152 `im_post` (expand_boxes bbox/bbox_transform.py:365-381 -> int32 boxes,
 *           (M+2)x(M+2) zero-padded mask -> cv2.resize -> > 0.5 -> paste into [H,W] -> pycocotools.mask.encode), run by the
 *           reference on the host with numpy + cv2 + pycocotools for every detection.
 * mask_probs [n,C,M,M] fp32 (M <= 28; the plane of cls_inds[d] is used when C > 1, plane 0 otherwise), boxes [n,4]
 * (x1,y1,x2,y2 = pred_boxes[:,1:]), cls_inds int64 [n]; n_dev (optional device count <= n); image H <= 2048, W <= 2048.
 * counts [n][cap] uint32: the UNCOMPRESSED COCO run lengths of detection d (column-major, starting with the zeros run,
 * exactly maskApi.c rleEncode); run_len [n] their number (0 for d >= *n_dev); *overflow = 1 if some detection needs more
 * than cap counts (run_len then holds the needed size).  The compressed `counts` string of the COCO dict is a pure
 * function of these numbers (rleToString), applied on the host by upsnet_b200.operators.im_post.
 * Workspace: upsnet_im_post_workspace_bytes(n, cap). */
int upsnet_im_post_workspace_bytes(int n, int cap, size_t *bytes);
int upsnet_im_post_rle(const float *mask_probs, int C, int M, const float *boxes, const int64_t *cls_inds, int n,
                       const int *n_dev, int H, int W, uint32_t *counts, int cap, int *run_len, int *overflow,
                       void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------
 * Backward kernels of the custom operators (training configuration, BASELINE config #4).  fp32 NCHW, ONE image per call
 * for the deformable kernels (the reference loops over the batch: functions/deform_conv.py:84-104).
 *
 * upsnet_dcn_im2col:       col [Cin*kh*kw, Ho*Wo] = zero-padded bilinear samples (* mask)      -- d(weight) = dY * col^T
 *   replaces: operators/src/deform_conv_kernel.cu:194-242 (K1), mod_deform_conv_kernel.cu:187-249 (K4)
 * upsnet_dcn_col2im:       dx [Cin,H,W] (zeroed by the call) += bilinear weights * dcol (* mask)
 *   replaces: deform_conv_kernel.cu:293-343 (K2), mod_deform_conv_kernel.cu:251-308 (K5)
 * upsnet_dcn_col2im_coord: doffset [2*kh*kw, Ho*Wo] and, with a mask, dmask [kh*kw, Ho*Wo]
 *   replaces: deform_conv_kernel.cu:391-449 (K3), mod_deform_conv_kernel.cu:310-381 (K6)
 * x [Cin,H,W]; offset [2*kh*kw,Ho,Wo]; mask [kh*kw,Ho,Wo] (already activated) or NULL; deformable_groups = 1.
 */
int upsnet_dcn_im2col(const float *x, const float *offset, const float *mask, int Cin, int H, int W, int kh, int kw,
                      int stride_h, int stride_w, int pad_h, int pad_w, int dil_h, int dil_w, float *col, void *stream);
int upsnet_dcn_col2im(const float *dcol, const float *offset, const float *mask, int Cin, int H, int W, int kh, int kw,
                      int stride_h, int stride_w, int pad_h, int pad_w, int dil_h, int dil_w, float *dx, void *stream);
int upsnet_dcn_col2im_coord(const float *dcol, const float *x, const float *offset, const float *mask, int Cin, int H,
                            int W, int kh, int kw, int stride_h, int stride_w, int pad_h, int pad_w, int dil_h, int dil_w,
                            float *doffset, float *dmask, void *stream);

/* upsnet_roi_align_backward: dfeat [B,C,H,W] (zeroed by the call) += scatter of dout [R,C,PH,PW] to the bilinear taps.
 * replaces: operators/src/roi_align_kernel.cu:238-348 RoIAlignBackwardFeature (K8). */
int upsnet_roi_align_backward(const float *dout, const float *rois, int R, int B, int C, int H, int W, int PH, int PW,
                              int sampling_ratio, float spatial_scale, float *dfeat, void *stream);

/* ---------------------------------------------------------------------------------------
 * upsnet_rpn_targets: the RPN training targets of one image (training configuration, BASELINE config #4).
 * replaces: rpn/assign_anchor.py:447-595 _get_rpn_blobs, called per image by add_rpn_blobs (:370-445) from the data loaders
 *           (dataset/coco.py:129, cityscapes.py:122, ade20k.py:116): the float32 IoU matrix of the inside anchors against
 *           every box (the Cython bbox/bbox.pyx:21-65), its argmaxes and tie sets, two np.random.choice draws and four dense
 *           arrays per level, on the host.
 * Anchors: level l has field_sizes[l]^2 cells of A anchors, anchor (l, y, x, a) = float32(cell_anchors[l][a] (float64
 *   [L,A,4], generate_anchors.py:50-76) + (x, y, x, y) * strides[l]), ordered level, cell (y, x), a (generate_anchors.py:
 *   79-130).  Inside: in float64, x1 >= -straddle, y1 >= -straddle, x2 < im_width + straddle, y2 < im_height + straddle;
 *   every anchor when straddle_thresh < 0.
 * gt_boxes float32 [G,4], 1 <= G <= UPSNET_RPN_TARGETS_MAX_G (more: UPSNET_E_UNSUPPORTED).  IoU bit-exact to bbox.pyx as
 *   Cython compiles it (double `+ 1.0`, double `ua`).  fg = an inside anchor whose IoU equals some box's maximum over the
 *   inside anchors (a maximum of 0 included) or whose own maximum is >= positive_overlap; bg candidates = maximum <
 *   negative_overlap (float32 compares).  More than num_fg fg anchors: the ones drawn are disabled; then num_bg =
 *   batch_size - #fg anchors are drawn from the bg candidates (an fg anchor drawn becomes 0), and none is labelled 0 when
 *   there are no more than num_bg candidates.  A draw of `size` among n candidates takes the positions p (in anchor order)
 *   with the `size` smallest keys splitmix64(s ^ p * 0x9E3779B97F4A7C15), s = seed for the fg draw and splitmix64(seed)
 *   for the bg draw.
 * Outputs, the per-level blobs of the reference concatenated over levels: labels int64 [1,A,F,F] (-1 / 0 / 1),
 *   bbox_targets (bbox_transform_inv of the anchors with label 1 after the fg draw, against their first-argmax box),
 *   inside_weights (1 where the final label is 1) and outside_weights (float32(1.0 / #labels >= 0) where the label is
 *   >= 0), each float32 [1,4A,F,F] with channel a*4 + c; counts int32 [4] = inside anchors, fg candidates, final fg,
 *   final bg.  All device memory; the call never synchronises.
 * Workspace: upsnet_rpn_targets_workspace_bytes(total anchors, batch_size). */
#define UPSNET_RPN_TARGETS_MAX_G 4096
int upsnet_rpn_targets_workspace_bytes(long long num_anchors, int batch_size, size_t *bytes);
int upsnet_rpn_targets(const float *gt_boxes, int G, const double *cell_anchors, const int *strides,
                       const int *field_sizes, int L, int A, double im_height, double im_width, double straddle_thresh,
                       float positive_overlap, float negative_overlap, int batch_size, int num_fg, unsigned long long seed,
                       int64_t *labels, float *bbox_targets, float *inside_weights, float *outside_weights, int *counts,
                       void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------
 * upsnet_proposal_targets: the Mask R-CNN proposal targets of one image (training configuration).
 * replaces: operators/modules/proposal_mask_target.py:37-62 ProposalMaskTarget.forward, run in the middle of the model's
 *           forward (models/resnet_upsnet.py:105-110): rois.cpu(), add_proposals (dataset/json_dataset.py:335-348,
 *           454-516, 538-556), sample_rois (bbox/sample_rois.py:51-176), add_mask_rcnn_blobs with pycocotools' polygon
 *           rasteriser (mask/mask_transform.py:195-323) and nine host-to-device copies.
 * Rows: the G gt rows of the roidb entry, then rois[r, 1:] * float32(1 / im_scale) for the rows r with rois[r, 0] == 0
 *   (float32, as numpy >= 2 computes it).  A gt row takes max overlap / class / gt row from gt_max_overlaps,
 *   gt_max_classes (max / argmax of the entry's gt_overlaps; -1 / 0 for crowd) and gt_box_to_gt_ind; a proposal takes
 *   the IoU (bit-exact to the compiled bbox.pyx) against every gt row of class > 0, crowd included: with a first-argmax
 *   max > 0, (max, gt_classes of that row, that row), else (0, 0, -1).  Every gt row must have gt_classes > 0.
 * Sampling: fg = max >= fg_thresh (> 0), bg = bg_thresh_lo <= max < bg_thresh_hi (float32 compares); fg_per_image is
 *   int(np.round(fg_fraction * batch_rois)), computed by the caller; min(fg_per_image, #fg) fg rows and
 *   min(batch_rois - that, #bg) bg rows are drawn: a draw of `size` among n candidates takes the positions p (in row
 *   order) with the `size` smallest keys splitmix64(s ^ p * 0x9E3779B97F4A7C15), s = seed for the fg draw and
 *   splitmix64(seed) for the bg draw (the rule of upsnet_rpn_targets), and keeps them in row order.
 * Outputs (batch_rois rows; rows past the fg + bg rows are 0, nongt_inds past its count -1):
 *   rois_out float32 [batch_rois,5] = (0, box * im_scale); labels int64 [batch_rois] = class of the fg rows, 0 for bg;
 *   bbox_targets / bbox_inside_weights / bbox_outside_weights float32 [batch_rois, 4K]: at columns 4*label..4*label+3
 *   of an fg row, bbox_transform_inv(box, gt box of gt_inds[box_to_gt_ind]) with weights (wx, wy, ww, wh) multiplied
 *   first, and weights 1 (an fg proposal on a crowd box regresses to the crowd box); nongt_inds int64 [batch_rois] = the
 *   output rows that are proposals; roi_has_mask uint8 [batch_rois] = label > 0.
 *   Mask rows (capacity max(fg_per_image, 1)): mask_rois float32 [.,5] = the fg rows of rois_out; mask_int32 float32
 *   [., K * M * M], -1 outside the label's M x M block, which holds (row-major [y][x]) the union of the polygons of the
 *   non-crowd object whose box (obj_boxes: float32 min / max of its polygon coordinates) has the largest IoU with the
 *   row's box (first argmax), rasterised as maskApi.c rleFrPoly does at M x M after ((p - x1) * M) / max(x2 - x1, 1) in
 *   float32.  Without fg rows: one mask row, the first bg row, all -1, and roi_has_mask[0] = 1.
 *   Objects: obj_poly_off [num_objects + 1] indexes polygons, poly_vert_off [P + 1] indexes verts float32 [V,2].
 *   counts int32 [5] = fg rows, bg rows, mask rows, error (1 when there is neither fg nor bg: the reference raises
 *   IndexError), nongt_inds count.  All device memory; the call never synchronises.
 * Limits: 1 <= G <= UPSNET_RPN_TARGETS_MAX_G, mask_size <= 32, batch_rois <= 4096, cls_agnostic_bbox_reg = 0; otherwise
 *   UPSNET_E_UNSUPPORTED.  Workspace: upsnet_proposal_targets_workspace_bytes(R, G, batch_rois). */
int upsnet_proposal_targets_workspace_bytes(int num_rois, int num_gt, int batch_rois, size_t *bytes);
int upsnet_proposal_targets(const float *rois, int R, const float *gt_boxes, const float *gt_max_overlaps,
                            const int *gt_max_classes, const int *gt_classes, const int *gt_box_to_gt_ind, int G,
                            const float *obj_boxes, const int *obj_poly_off, const int *poly_vert_off, const float *verts,
                            int num_objects, float im_scale, int num_classes, int batch_rois, int fg_per_image,
                            float fg_thresh, float bg_thresh_hi, float bg_thresh_lo, float wx, float wy, float ww,
                            float wh, int cls_agnostic_bbox_reg, int mask_size, unsigned long long seed, float *rois_out,
                            int64_t *labels, float *bbox_targets, float *bbox_inside_weights,
                            float *bbox_outside_weights, int64_t *nongt_inds, float *mask_rois, float *mask_int32,
                            unsigned char *roi_has_mask, int *counts, void *workspace, size_t workspace_bytes,
                            void *stream);

/* ---------------------------------------------------------------------------------------
 * upsnet_panoptic_loss_forward / _backward: the panoptic head of the training forward of one image, fused.
 * replaces: models/resnet_upsnet.py:156-179 and 250-257: the class gather of mask_score, SegTerm and MaskTerm
 *           (operators/modules/unary_logits.py:24-105), the void logits, torch.cat, MaskMatching
 *           (operators/modules/mask_matching.py:37-58), calc_panoptic_acc and
 *           CrossEntropyLoss(ignore_index=255, reduce=False)(...).mean(), with autograd's backward of that composition.
 *           No [1,k,h,w] plane is built; backward keeps 8 bytes per pixel.
 * Inputs (device): fcn_score float32 [S,h,w]; mask_score float32 [k,C,M,M], C == num_classes or C == 1 (already
 *   gathered); gt_rois float32 [k,5] = (0,x1,y1,x2,y2); cls_idx int64 [k] (a value outside 0..num_classes-1 is treated
 *   as 0); seg_gt int64 [h,w]; mask_gt [G,h,w], uint8 or int64 (mask_gt_is_int64); keep_inds int64 [k] or NULL (then
 *   G == k; an index outside 0..G-1 paints nothing).  num_stuff = S - num_classes + 1; thing class c is seg channel
 *   T(c) = num_stuff + c - 1.
 * Channels at a pixel: 0..num_stuff-1 = fcn_score; num_stuff + i = seg_i + mask_i; with enable_void a last channel
 *   max over t >= num_stuff of fcn_score[t], minus max over i of seg_i (the zeros outside the windows take part).
 *   seg_i = fcn_score[T(cls_i)] inside SegTerm's window, else 0: with b = float32(roi) * box_scale,
 *     [int(b.y1), int(rint(b.y2) + 1)) x [int(b.x1), int(rint(b.x2) + 1)), rint = half to even, bounds clamped to the
 *     image (a negative bound is clamped to 0, where the reference's slice would wrap around); empty for class 0.
 *   mask_i = mask_score[i, cls_i] (channel 0 when C == 1) resized to (bh,bw) = (max(r.y2-r.y1+1,1), max(r.x2-r.x1+1,1)),
 *     r = trunc(b), by ATen's bilinear rule (align_corners = False: src = max(scale * (dst + 0.5) - 0.5, 0) with
 *     scale = M / bw in float32, second tap min(i0 + 1, M - 1)), pasted at (r.y1, r.x1), cropped to the image, else 0.
 * Ground truth at a pixel: seg_gt where it is <= S - num_classes or >= 255, else -1; then num_stuff + j for the last j
 *   with mask_gt[keep_inds[j]] (mask_gt[j] without keep_inds) neither 0 nor 255; what is still -1 becomes num_stuff + k
 *   with keep_inds, 255 without.  A value that is neither a channel nor 255 (the reference's cross-entropy raises on
 *   it) gives no loss and no gradient and is never counted correct.
 * Outputs (device): loss[1] = sum of (log-sum-exp - logit of the ground-truth channel) over the pixels whose ground
 *   truth is not 255, divided by h*w; accuracy[1] = counts[0] / (h*w - counts[1]); counts int32 [2] = pixels whose
 *   arg-max channel (ties: the lowest) equals the ground truth, pixels whose ground truth is 255; lse float32 [h*w] and
 *   gt_channel int32 [h*w] are what backward reads.  When every pixel is 255 the accuracy is 0 / 0 (the reference
 *   asserts there).
 * Backward: grad_out float32 [1] on the device; d_fcn_score float32 [S,h,w] (every element written) and d_mask_score
 *   float32 [k,C,M,M] (zero outside the selected channel); either may be NULL.  With p = softmax and
 *   g_c = (p_c - [c == gt]) * grad_out / (h*w) on the pixels with a loss: stuff channels get g_c; T(c) gets the g of
 *   the instances of class c whose SegTerm window covers the pixel, + g_void on the arg-max thing channel, - g_void on
 *   the channel of the instance that wins max_i seg_i (nothing when a zero wins); d_mask_score is the transpose of the
 *   resize-and-paste applied to g_{num_stuff+i}, computed as a gather.
 * Same inputs give the same bytes (no atomics); no call synchronises or reads the device; both are capturable.
 * Limits: M <= 32, S*h*w < 2^31, k*C*M*M < 2^31 (else UPSNET_E_UNSUPPORTED); k >= 1.
 * Workspace: upsnet_panoptic_loss_workspace_bytes(k, h, w), for either call; nothing in it outlives the call. */
int upsnet_panoptic_loss_workspace_bytes(int k, int h, int w, size_t *bytes);
int upsnet_panoptic_loss_forward(const float *fcn_score, int S, int h, int w, const float *mask_score, int k, int C,
                                 int mask_size, const float *gt_rois, const int64_t *cls_idx, const int64_t *seg_gt,
                                 const void *mask_gt, int mask_gt_is_int64, int G, const int64_t *keep_inds,
                                 int num_classes, int enable_void, float box_scale, float *loss, float *accuracy,
                                 int *counts, float *lse, int *gt_channel, void *workspace, size_t workspace_bytes,
                                 void *stream);
int upsnet_panoptic_loss_backward(const float *fcn_score, int S, int h, int w, const float *mask_score, int k, int C,
                                  int mask_size, const float *gt_rois, const int64_t *cls_idx, int num_classes,
                                  int enable_void, float box_scale, const float *lse, const int *gt_channel,
                                  const float *grad_out, float *d_fcn_score, float *d_mask_score, void *workspace,
                                  size_t workspace_bytes, void *stream);

/* upsnet_panoptic_gt: the ground-truth rule above alone (MaskMatching.forward), as the int64 [h,w] map the reference
 * returns; k counts keep_inds and is ignored without them. */
int upsnet_panoptic_gt(const int64_t *seg_gt, const void *mask_gt, int mask_gt_is_int64, int G, const int64_t *keep_inds,
                       int k, int h, int w, int num_seg_classes, int num_classes, int64_t *panoptic_gt, void *stream);

/* upsnet_draw_keys: keys[p] = the draw key of candidate position p = 0..n-1 (the rule of upsnet_rpn_targets: stream_id
 * 0 is its fg draw, 1 its bg draw), so that a host restatement of the rule can be compared with the device's. */
int upsnet_draw_keys(unsigned long long seed, int stream_id, int n, unsigned long long *keys, void *stream);

/* ---- training losses (train_loss.cu) ----------------------------------------------------
 * upsnet_semantic_loss_forward / _backward: the semantic head's loss of one image, with the x4 up-sampling fused in.
 * replaces: models/fcn.py:101 F.interpolate(fcn_score, None, 4, mode='bilinear', align_corners=False) and
 *           models/resnet_upsnet.py:79,131 CrossEntropyLoss(ignore_index=255)(fcn_output, seg_gt), with autograd's
 *           backward of that composition.  No [S,4h,4w] tensor is built; backward keeps 4 bytes per output pixel.
 * Inputs (device): fcn_score float32 [S,h,w]; seg_gt [4h,4w], uint8 or int64 (seg_gt_is_int64).  The logits of output
 *   pixel o are those upsnet_upsample_bilinear_nchw (factor 4) writes, bit for bit (up4.cuh).  t(o) = seg_gt[o].
 * Outputs (device): loss[1] = sum over pixels with t in 0..S-1 of (log-sum-exp - logit of t), divided by their count N
 *   (NaN when N = 0, as torch's mean); counts int32 [2] = (N, pixels whose label is neither 255 nor in 0..S-1: torch
 *   would assert on them; here they give no loss and no gradient and are not in N); lse float32 [4h*4w], 16-byte
 *   aligned, is what backward reads (written everywhere, meaningful where t is a channel).
 * Backward: grad_out float32 [1] and counts (forward's) on the device; d_fcn_score float32 [S,h,w], every element
 *   written: grad_out / N * sum over o of w(o -> source) * (softmax_c(o) - [c = t(o)]), w the up-sampling's tap
 *   weights, as a gather (no atomics); all zeros when N = 0.
 * Same inputs give the same bytes; no call synchronises or reads the device; both are capturable.
 * Limits: S*h*w < 2^31, 16*h*w < 2^31, S <= 32767 (else UPSNET_E_UNSUPPORTED).
 * Workspace: upsnet_semantic_loss_workspace_bytes(h, w), forward only; nothing in it outlives the call. */
int upsnet_semantic_loss_workspace_bytes(int h, int w, size_t *bytes);
int upsnet_semantic_loss_forward(const float *fcn_score, int S, int h, int w, const void *seg_gt, int seg_gt_is_int64,
                                 float *loss, int *counts, float *lse, void *workspace, size_t workspace_bytes,
                                 void *stream);
int upsnet_semantic_loss_backward(const float *fcn_score, int S, int h, int w, const void *seg_gt, int seg_gt_is_int64,
                                  const float *lse, const int *counts, const float *grad_out, float *d_fcn_score,
                                  void *stream);

/* upsnet_fcn_roi_loss_forward / _backward: the semantic head's ROI loss of one image (train.fcn_with_roi_loss).
 * replaces: models/fcn.py:102-106 roi_score = score(RoIAlign(M, M, spatial_scale)(feat, rois)), feat the 512-channel
 *           concat of the four up-sampled levels, and models/resnet_upsnet.py:132-134
 *           CrossEntropyLoss(ignore_index=255, reduce=False)(roi_score, seg_roi_gt).mean(), with autograd's backward.
 *           The score conv and ROIAlign commute, so the loss samples the S-plane fcn_score (the score conv's output,
 *           bias included) instead: neither feat, the [R,512,M,M] roi features nor their gradients are built.
 * Inputs (device): fcn_score float32 [S,h,w]; bias float32 [S] (the score conv's); rois float32 [R,5] in image
 *   coordinates (column 0, the batch index, is not read: one image); seg_roi_gt [R,M,M], uint8 or int64
 *   (seg_roi_gt_is_int64).  The roi score of cell (r, ph, pw), channel c, is ROIAlign of plane c by the forward rule of
 *   upsnet_roi_align_forward (roi_sample.cuh, aligned=False, sampling_ratio x sampling_ratio samples) plus
 *   bias[c] * (1 - n_inside / count): ROIAlign gives a sample outside the map 0, so sampling fcn_score carries only
 *   n_inside / count of the bias that the reference adds once per cell.  The term is 0 for every cell whose samples are
 *   inside the map.
 * Outputs (device): loss[1] = sum over cells whose target t is in 0..S-1 of (log-sum-exp - roi score of t), divided by
 *   R*M*M (reduce=False then mean: ignored cells count in the denominator); counts int32 [2] = (cells with a target,
 *   cells whose target is neither 255 nor in 0..S-1: no loss and no gradient); lse float32 [R*M*M], what backward reads.
 * Backward: lse (forward's) and grad_out float32 [1] on the device; d_fcn_score float32 [S,h,w], every element written
 *   (0 where no roi samples): the transpose of the sampling applied to (softmax - onehot) * grad_out / (R*M*M), as a
 *   gather over the rois in order with the forward's tap weights; d_bias float32 [S], the gradient of the correction
 *   term alone (the caller adds it to what the bias receives through fcn_score).  No atomics.
 * Same inputs give the same bytes; no call synchronises or reads the device; both are capturable.
 * Limits: 1 <= R <= 1024, M <= 64, sampling_ratio = 2, S*h*w < 2^31, S*R*M*M < 2^31, S <= 32767 (else
 *   UPSNET_E_UNSUPPORTED, before any launch).
 * Workspace: upsnet_fcn_roi_loss_workspace_bytes(S, R, M, backward) (UPSNET_E_UNSUPPORTED for R or M beyond the
 *   limits): backward = 0 for the forward's (block partials), 1 for the backward's (4*S*R*M*M bytes of roi-score gradient plus 4*R*M*M); nothing in it outlives the call. */
int upsnet_fcn_roi_loss_workspace_bytes(int S, int R, int M, int backward, size_t *bytes);
int upsnet_fcn_roi_loss_forward(const float *fcn_score, const float *bias, int S, int h, int w, const float *rois, int R,
                                const void *seg_roi_gt, int seg_roi_gt_is_int64, int M, int sampling_ratio,
                                float spatial_scale, float *loss, int *counts, float *lse, void *workspace,
                                size_t workspace_bytes, void *stream);
int upsnet_fcn_roi_loss_backward(const float *fcn_score, const float *bias, int S, int h, int w, const float *rois, int R,
                                 const void *seg_roi_gt, int seg_roi_gt_is_int64, int M, int sampling_ratio,
                                 float spatial_scale, const float *lse, const float *grad_out, float *d_fcn_score,
                                 float *d_bias, void *workspace, size_t workspace_bytes, void *stream);

/* upsnet_rpn_loss_forward / _backward: the RPN loss of one image over all FPN levels in one launch.
 * replaces: models/rpn.py:60-92 RPNLoss.forward (with_fpn): per level, the [:, :, :h, :w] slices of the label maps,
 *           F.binary_cross_entropy_with_logits(score, label, weight = label != -1, reduction='sum') / rpn_batch_size
 *           and smooth_l1_loss(sigma = 3) / batch (= 1), summed over the levels; with autograd's backward.
 * Inputs: host arrays of num_levels entries (num_levels <= 8): h[l], w[l] = the score map's size; device pointers
 *   cls_score[l] float32 [A,h,w], bbox_pred[l] float32 [4A,h,w] (contiguous); labels[l] int64 and bbox_targets[l],
 *   bbox_inside_weights[l], bbox_outside_weights[l] float32, read in place from fields at least as large as the map:
 *   element (c, y, x) of level l is at c * strides[2l] + y * strides[2l+1] + x (label_strides for the labels,
 *   bbox_strides for the three box fields), no slice copies.
 * Outputs (device): cls_loss[1] = sum over anchors with label != -1 of (1 - t) x + m + log(exp(-m) + exp(-x - m)),
 *   m = max(-x, 0), divided by rpn_batch_size; bbox_loss[1] = sum of ow * (|d| < 1/9 ? 4.5 d^2 : |d| - 0.5/9),
 *   d = iw * (pred - target).
 * Backward: grad_cls, grad_bbox float32 [1] on the device; d_cls_score[l] = (label != -1) (sigmoid(x) - t) grad_cls /
 *   rpn_batch_size, d_bbox_pred[l] = ow iw (|d| < 1/9 ? 9 d : sign d) grad_bbox, every element written; either host
 *   array may be NULL.
 * Same inputs give the same bytes; no call synchronises or reads the device; both are capturable.  Batch size 1.
 * Limits: num_levels <= 8, 4A*h*w < 2^31 per level and A * sum h*w < 2^31 (else UPSNET_E_UNSUPPORTED).
 * Workspace: upsnet_rpn_loss_workspace_bytes(A * sum of h[l]*w[l]), forward only. */
int upsnet_rpn_loss_workspace_bytes(int num_anchors, size_t *bytes);
int upsnet_rpn_loss_forward(int num_levels, int A, const int *h, const int *w, const float *const *cls_score,
                            const float *const *bbox_pred, const int64_t *const *labels, const long long *label_strides,
                            const float *const *bbox_targets, const float *const *bbox_inside_weights,
                            const float *const *bbox_outside_weights, const long long *bbox_strides,
                            float rpn_batch_size, float *cls_loss, float *bbox_loss, void *workspace,
                            size_t workspace_bytes, void *stream);
int upsnet_rpn_loss_backward(int num_levels, int A, const int *h, const int *w, const float *const *cls_score,
                             const float *const *bbox_pred, const int64_t *const *labels, const long long *label_strides,
                             const float *const *bbox_targets, const float *const *bbox_inside_weights,
                             const float *const *bbox_outside_weights, const long long *bbox_strides,
                             float rpn_batch_size, const float *grad_cls, const float *grad_bbox,
                             float *const *d_cls_score, float *const *d_bbox_pred, void *stream);

/* upsnet_mask_rcnn_loss_forward / _backward: the Mask R-CNN loss and accuracy of one image.
 * replaces: models/rcnn.py:159-197 MaskRCNNLoss.forward: CrossEntropyLoss(ignore_index=-1), smooth_l1_loss(sigma = 1)
 *           / R, rcnn_accuracy and mask_loss / (mask_weight.sum() + 1e-10); with autograd's backward.
 * Inputs (device, contiguous): cls_score float32 [R,K]; cls_label int64 [R]; bbox_pred, bbox_target,
 *   bbox_inside_weight, bbox_outside_weight float32 [R,B]; mask_score, mask_target float32 of mask_numel elements
 *   each ([n,K,M,M] and [n,K*M*M]; both may be NULL when mask_numel = 0).  Forward reads each once.
 * Outputs (device): cls_loss[1] = mean over rows with a label in 0..K-1 of (log-sum-exp - logit of the label) (NaN
 *   without such rows); bbox_loss[1] = sum of ow * (|d| < 1 ? d^2 / 2 : |d| - 1/2), d = iw * (pred - target), / R;
 *   mask_loss[1] = sum over t != -1 of -x (t - b) + log(1 + exp(-|x|)), b = (x >= 0), divided by float32(W) + 1e-10
 *   in float32, W the number of such elements (0 when W = 0); accuracy[1] = (counts[2] - counts[1]) / (R - counts[1])
 *   (rcnn_accuracy as written: the rows labelled -1 are subtracted from the correct ones too); counts int32 [4] =
 *   (rows with a label in 0..K-1, rows labelled -1, rows whose arg-max (ties: the lowest class) equals the label, W).
 *   A label outside -1..K-1 (torch asserts on it) gives no loss and no gradient.
 * Backward: counts (forward's) and grad_cls, grad_bbox, grad_mask float32 [1] on the device; d_cls_score =
 *   (softmax - onehot) grad_cls / counts[0] on rows with a label, else 0; d_bbox_pred = ow iw (|d| < 1 ? d : sign d)
 *   grad_bbox / R; d_mask_score = (t != -1) (sigmoid(x) - t) grad_mask / (float32(W) + 1e-10).  Every element is
 *   written; any of the three may be NULL.
 * Same inputs give the same bytes; no call synchronises or reads the device; both are capturable.
 * Limits: R*K, R*B and mask_numel < 2^31 (else UPSNET_E_UNSUPPORTED); R >= 1.
 * Workspace: upsnet_mask_rcnn_loss_workspace_bytes(R, B, mask_numel), forward only. */
int upsnet_mask_rcnn_loss_workspace_bytes(int R, int B, long long mask_numel, size_t *bytes);
int upsnet_mask_rcnn_loss_forward(const float *cls_score, const int64_t *cls_label, int R, int K, const float *bbox_pred,
                                  const float *bbox_target, const float *bbox_inside_weight,
                                  const float *bbox_outside_weight, int B, const float *mask_score,
                                  const float *mask_target, long long mask_numel, float *cls_loss, float *bbox_loss,
                                  float *mask_loss, float *accuracy, int *counts, void *workspace,
                                  size_t workspace_bytes, void *stream);
int upsnet_mask_rcnn_loss_backward(const float *cls_score, const int64_t *cls_label, int R, int K, const float *bbox_pred,
                                   const float *bbox_target, const float *bbox_inside_weight,
                                   const float *bbox_outside_weight, int B, const float *mask_score,
                                   const float *mask_target, long long mask_numel, const int *counts,
                                   const float *grad_cls, const float *grad_bbox, const float *grad_mask,
                                   float *d_cls_score, float *d_bbox_pred, float *d_mask_score, void *stream);

/* ---- panoptic training labels (labels.cu) ----
 * upsnet_training_labels: the label maps of one training image (the label block of the reference's Cityscapes / COCO
 * loaders and collate / gt_list_to_blob) from its uint8 label map [h0,w0]:
 *   seg_gt     int64 [Hs,Ws]     = label[seg_rows[y], seg_cols[x]]
 *   seg_gt_4x  int64 [Hq,Wq]     = label[q_rows[y], q_cols[x]]
 *   seg_roi_gt int64 [n_roi,M,M] = label[roi_rows[i*M + y], roi_cols[i*M + x]]
 *   mask_gt    uint8 or int64 [G,Hm,Wm] = 1 where canvas pixel (m_rows[y], m_cols[x]) is set by Pillow's polygon fill
 *              (ImageDraw.polygon(outline=1, fill=1)) of any polygon of instance g, else 0
 * Every table is int32 and host-built (cv2 INTER_NEAREST composed through each resize, the flip folded into the
 * label-map columns); -1 marks padding, written as 255.  m_cols is non-decreasing on its non-negative entries.
 * Polygons: instance g owns polygons [obj_poly[g], obj_poly[g+1]), polygon p the int32 (x, y) vertex pairs
 * [poly_vert[p], poly_vert[p+1]) of verts, already truncated toward zero as Pillow does; obj_yrange[2g..2g+1] is the
 * instance's lowest and highest vertex y.  max_poly_verts / max_obj_verts are the largest vertex counts of one polygon
 * and of one instance: above the limits below, or G above UPSNET_LABELS_MAX_G, the call returns UPSNET_E_UNSUPPORTED
 * before any launch.  One owner thread per output element, no atomics: the same inputs give the same bytes. */
#define UPSNET_LABELS_MAX_POLY_VERTS 1024
#define UPSNET_LABELS_MAX_OBJ_VERTS 1536
#define UPSNET_LABELS_MAX_G 65535
int upsnet_training_labels(const unsigned char* label, int h0, int w0, const int* seg_rows, int Hs, const int* seg_cols,
                           int Ws, int64_t* seg_gt, const int* q_rows, int Hq, const int* q_cols, int Wq,
                           int64_t* seg_gt_4x, const int* m_rows, int Hm, const int* m_cols, int Wm, const int* obj_poly,
                           const int* poly_vert, const int* verts, const int* obj_yrange, int G, int max_poly_verts,
                           int max_obj_verts, void* mask_gt, int mask_gt_is_int64, const int* roi_rows,
                           const int* roi_cols, int n_roi, int M, int64_t* seg_roi_gt, void* stream);

/* ---- optimiser step (sgd.cu) ----------------------------------------------------------------
 * upsnet_sgd_apply: one momentum-SGD step over every parameter listed in a chunk table, in one launch.
 * replaces: lib/nn/optimizer.py:80-104 SGD.step(lr) (four element-wise ops per parameter, issued from Python), the
 *           '/ world' and copy into p.grad of an all-reduced bf16 bucket before it, and the momentum decay of
 *           upsnet_end2end_train.py:235-240 (every momentum buffer .div_(10) after a decay iteration).
 * Chunk table (device, 8-byte aligned, num_chunks entries of upsnet_sgd_chunk): one CTA per entry.  param / buf / grad
 *   point at the entry's first element; n >= 0 elements; group indexes the three host arrays of num_groups entries
 *   (1 <= num_groups <= UPSNET_SGD_MAX_GROUPS, else UPSNET_E_UNSUPPORTED).  kind UPSNET_SGD_GRAD_F32: grad is float32
 *   (a p.grad); UPSNET_SGD_GRAD_BF16: grad is a bf16 bucket segment, read as float32 and multiplied by inv_world
 *   (= 1.0f / world, what torch's CUDA true division by a host scalar does); UPSNET_SGD_GRAD_NONE: a parameter with a
 *   momentum buffer but no gradient this step, whose buffer only the decay touches (grad unused).  buf may be NULL in a
 *   group whose momentum is 0.  Any addresses are accepted: 16-byte accesses are used where param, buf and grad allow
 *   them (grad: 16 bytes for float32, 8 for bf16), element accesses otherwise.  Entries of at most UPSNET_SGD_CHUNK
 *   elements keep the grid balanced; the ranges of different entries must not overlap.
 * Learning rate: lr_table == NULL: `lr`, no decay (the drop-in step(lr)).  Otherwise the scheduled step: k =
 *   *iteration - table_begin (device int), lr = lr_table[k] (device float64 [table_len]) and decay = decay_table[k]
 *   (device uint8); when k is outside [0, table_len) the launch changes nothing.
 * Rounding, per element, with glr = group_lr[group], wd = group_weight_decay[group], m = group_momentum[group]; each line
 *   rounds once to float32 (fma: one fused rounding; torch's CUDA add_(x, alpha=) is self + alpha * x, one FMA):
 *     d = g                              (bf16: float(g) * inv_world)
 *     d = fma(wd, p, d)                  only if wd != 0 (skipped, not multiplied by 0)
 *     a = (float)(glr * lr)              the double product rounded once, as torch converts the Python scalar
 *     b = fma(a, d, b * m); p = p - b    if m != 0 (a new buffer is +0, so its first value is +0 * m + a d)
 *     p = p - d                          if m == 0: lr does not enter, as in the reference
 *     b = b * 0.1f                       after the update, on a decay step (div_(10) on CUDA multiplies by 1.0f / 10)
 *   p.grad is not written (the reference leaves g + wd p in it; nothing reads that).  No atomics: same inputs, same bytes.
 * upsnet_sgd_pack: the bf16 bucket of FlatBucketAllReduce.start() from the parameters' float32 gradients, one launch per
 *   bucket: out[i] = bf16 round-to-nearest-even of grad[i] (torch's .to(torch.bfloat16)), zeros where grad is NULL (a
 *   None gradient).  Table (device, 8-byte aligned) of upsnet_sgd_pack_chunk, one CTA per entry, any alignment.
 * upsnet_sgd_advance: *iteration += 1 in a one-thread launch; the scheduled step issues it after its apply launches.
 * None of the three synchronises or reads the device; all are capturable in a CUDA graph. */
#define UPSNET_SGD_MAX_GROUPS 16
#define UPSNET_SGD_CHUNK 8192
#define UPSNET_SGD_GRAD_F32 0
#define UPSNET_SGD_GRAD_BF16 1
#define UPSNET_SGD_GRAD_NONE 2
typedef struct {
  float *param;
  float *buf;
  const void *grad;
  int n;
  int group;
  int kind;
  float inv_world;
} upsnet_sgd_chunk; /* 40 bytes */
typedef struct {
  const float *grad;
  void *out;
  int n;
  int reserved;
} upsnet_sgd_pack_chunk; /* 24 bytes */
int upsnet_sgd_apply(const upsnet_sgd_chunk *chunks, int num_chunks, int num_groups, const double *group_lr,
                     const float *group_weight_decay, const float *group_momentum, double lr, const double *lr_table,
                     const unsigned char *decay_table, const int *iteration, int table_begin, int table_len,
                     void *stream);
int upsnet_sgd_pack(const upsnet_sgd_pack_chunk *chunks, int num_chunks, void *stream);
int upsnet_sgd_advance(int *iteration, void *stream);

/* ---- dense convolution / FC backward (conv_backward.cu) ------------------------------------------
 * For a layer y = act(conv(x, W) + b [+ residual]) run by upsnet_igemm_forward, the gradients of x, W, b and the
 * residual from dY.  replaces: autograd's conv backward (cuDNN dgrad / wgrad and the bias / residual reductions) of the
 * trainable nn.Conv2d, nn.Linear and nn.ConvTranspose2d layers of models/resnet.py, models/fpn.py, models/rpn.py and
 * models/rcnn.py.  None of these synchronises or reads the device; all are capturable in a CUDA graph.  No atomics: the
 * same inputs give the same bytes.  precision is UPSNET_PREC_BF16X3 (g and x stored as hi/lo pairs) or UPSNET_PREC_BF16.
 *
 * upsnet_conv_grad_prepare: dy float32 logical [N,C,H,W], stored NCHW, or NHWC with UPSNET_GRAD_DY_NHWC (contiguous
 *   either way).  g = dy * [y > 0] with UPSNET_GRAD_RELU (y float32 NHWC [N,H,W,Cg], the forward's output), else dy,
 *   written NHWC [N,H,W,Cp] with Cp = Cg rounded up to a multiple of 64 and zeros in the padding: bf16 (PREC_BF16) or a
 *   pair [N,H,W,2 Cp] (PREC_BF16X3, UPSNET_DTYPE_PAIR layout).  Cg = C, or 4 C with UPSNET_GRAD_UNSHUFFLE2: then dy is
 *   [N,C,2H,2W] (the output of a ConvTranspose2d(k = 2, s = 2)) and g[n,h,w,(2a + b) C + c] = dy[n,c,2h + a,2w + b], the
 *   gradient of the 1x1 conv to 4 C channels that the engine makes of it.  dbias (may be NULL): float32 [C], the sum of g
 *   over the pixels (and the four (a, b) groups), accumulated in fp64 in a fixed order and rounded once; needs a
 *   workspace of upsnet_conv_grad_prepare_workspace_bytes.  dres (may be NULL; not with UNSHUFFLE2): float32 NHWC
 *   [N,H,W,C] = g, or with UPSNET_GRAD_RES_UP2 (H, W even) [N,H/2,W/2,C] = the sum of g over each 2x2 block,
 *   ((g00 + g01) + g10) + g11, the gradient of the nearest-neighbour up-sampled residual of the FPN top-down path.
 * upsnet_igemm_pack_weight_dgrad: the weights of the data gradient, for upsnet_igemm_forward run on g: W'[ci][tap][co] =
 *   W[co][ci][kh*kw - 1 - tap] as bf16 hi / lo planes [cout_pad(Cin)][kh*kw][Cp] (upsnet_igemm_pack_weight's format for
 *   a layer Cp -> Cin).  dX of a stride-1 layer is then upsnet_igemm_forward(g, ..., Cin = Cp, Cout = Cin, the same k and
 *   dilation, padding d (k - 1) - p) with a float32 NHWC output.
 * upsnet_conv_dgrad_scatter2: dX float32 NHWC [N,H,W,C] of a stride-2 1x1 layer (pad 0) from dxc = W^T g [N,(H+1)/2,
 *   (W+1)/2,C] (upsnet_igemm_forward of g with the 1x1 dgrad weights): dxc at the even pixels, 0 elsewhere.  C % 4 == 0.
 * upsnet_conv_wgrad: dw float32 [Cout][Cin][kh][kw] (torch's layout) = sum over the output pixels p and images of
 *   g[p][co] * x[p * stride + tap * dil - pad][ci] with x outside the image 0; x NHWC bf16 [N,H,W,Cin] or pair
 *   [N,H,W,2 Cin], g as upsnet_conv_grad_prepare writes it.  bf16x3: lo*hi + hi*lo + hi*hi products per pixel, bf16:
 *   hi*hi; fp32 accumulation in wgmma, K split over CTAs into fp32 partial tiles added in a fixed order.  With
 *   UPSNET_GRAD_UNSHUFFLE2 (1x1, Cout = 4 C) dw is written as the ConvTranspose2d weight [Cin][C][2][2] instead.
 *   Workspace: upsnet_conv_wgrad_workspace_bytes.  UPSNET_E_UNSUPPORTED before any launch for stride > 1 with k > 1
 *   or padding, Cin % 64 != 0, or kh * kw > 49 (groups != 1 has no parameter: it is not supported).
 */
#define UPSNET_GRAD_RELU 1
#define UPSNET_GRAD_RES_UP2 2
#define UPSNET_GRAD_UNSHUFFLE2 4
#define UPSNET_GRAD_DY_NHWC 8
int upsnet_conv_grad_prepare_workspace_bytes(int N, int C, int H, int W, int flags, size_t *bytes);
int upsnet_conv_grad_prepare(const float *dy, const float *y, void *g, float *dbias, float *dres, int N, int C, int H,
                             int W, int flags, int precision, void *workspace, size_t workspace_bytes, void *stream);
int upsnet_igemm_packed_weight_dgrad_bytes(int Cout, int Cin, int kh, int kw, size_t *bytes);
int upsnet_igemm_pack_weight_dgrad(const float *weight, int Cout, int Cin, int kh, int kw, void *packed, void *stream);
int upsnet_conv_dgrad_scatter2(const float *dxc, float *dx, int N, int H, int W, int C, void *stream);
int upsnet_conv_wgrad_workspace_bytes(int N, int H, int W, int Cin, int Cout, int kh, int kw, int stride_h, int stride_w,
                                      int pad_h, int pad_w, int dil_h, int dil_w, int precision, size_t *bytes);
int upsnet_conv_wgrad(const void *x_nhwc, const void *g, float *dw, int N, int H, int W, int Cin, int Cout, int kh, int kw,
                      int stride_h, int stride_w, int pad_h, int pad_w, int dil_h, int dil_w, int flags, int precision,
                      void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------
 * GroupNorm (csrc/group_norm.cu): nn.GroupNorm(groups, C) semantics -- biased variance, y = (x - mean) / sqrt(var + eps)
 * * gamma + beta -- over NHWC activations.  Deterministic: no atomics, fixed merge orders.
 * replaces: nn.GroupNorm(32, C) of models/fpn.py:43-58, rpn.py:37-40, rcnn.py:50-56 and :102-104, fcn.py:49-50.
 *
 * upsnet_group_norm_forward: whole maps.  x, y [N,H,W,C] in dtype (F32, BF16, or PAIR: [N,H,W,2C]); statistics cover
 * all H*W pixels of an image.  Three launches: per-(image, group, CTA) partial (count, mean, M2), their merge by Chan's
 * formula into stats[N][groups][2] = (mean, 1/sqrt(var + eps)) (fp32, caller-owned, read by the backward), and the
 * apply.  shift (fp32 [N][C] or NULL) is added after beta; flags: UPSNET_EPI_RELU; UPSNET_EPI_RES_UP2 with residual
 * [N,H/2,W/2,C] in dtype, read with nearest 2x up-sampling -- or, adding UPSNET_EPI_RES_BILINEAR, with the four
 * bilinear taps of upsnet_upsample2_bilinear_nhwc -- and added before the ReLU (H, W even).  C <= 1024 with
 * min(C, 256) dividing both 256 and C, else UPSNET_E_UNSUPPORTED.  Workspace: upsnet_group_norm_workspace_bytes.
 *
 * upsnet_group_norm_rows: R rows of HW pixels x C channels (NHWC, dtype as above), each row normalised on its own (the
 * mask branch's 14x14 roi maps, RCNN fc6 as [R,1024,1,1]); one launch, one warp per (row, group), two passes.  flags:
 * UPSNET_EPI_RELU.  n_dev (int32 device scalar or NULL): rows >= *n_dev are skipped and their output is unspecified.
 *
 * upsnet_group_norm_backward: gradients of y = act(GN(x) + shift [+ up2(residual)]), fp32 NHWC.  dy, x, dx [N,H,W,C];
 * y the forward output (read for the ReLU mask; pass it iff flags has UPSNET_EPI_RELU); stats from the forward.
 * dgamma, dbeta [C], dshift [N][C] (= per-image dbeta) and dres [N,H/2,W/2,C] (needs UPSNET_EPI_RES_UP2; with
 * UPSNET_EPI_RES_BILINEAR too it is the bilinear adjoint of the masked dy, as upsnet_upsample2_bilinear_nhwc_adjoint,
 * which needs C % 4 == 0) are each optional.  Workspace: upsnet_group_norm_backward_workspace_bytes. */
int upsnet_group_norm_workspace_bytes(int N, int C, int H, int W, int groups, size_t *bytes);
int upsnet_group_norm_forward(const void *x, const float *gamma, const float *beta, const float *shift,
                              const void *residual, void *y, float *stats, int N, int C, int H, int W, int groups,
                              float eps, int dtype, int flags, void *workspace, size_t workspace_bytes, void *stream);
int upsnet_group_norm_rows(const void *x, const float *gamma, const float *beta, void *y, int R, int C, int HW, int groups,
                           float eps, int dtype, int flags, const int *n_dev, void *stream);
int upsnet_group_norm_backward_workspace_bytes(int N, int C, int H, int W, int groups, size_t *bytes);
int upsnet_group_norm_backward(const float *dy, const float *x, const float *y, const float *stats, const float *gamma,
                               float *dx, float *dgamma, float *dbeta, float *dshift, float *dres, int N, int C, int H,
                               int W, int groups, int flags, void *workspace, size_t workspace_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* UPSNET_B200_H_ */
