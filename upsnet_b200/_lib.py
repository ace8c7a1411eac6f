"""ctypes binding of libupsnet_b200.so (the C ABI declared in include/upsnet_b200.h).

There is deliberately NO fallback: if the CUDA library cannot be loaded, or a tensor is not a
CUDA tensor, the ops raise.  (The reference does the same for non-CUDA tensors:
operators/functions/deform_conv.py:40-41, functions/roialign.py:34-35.)
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libupsnet_b200.so")
_lib = None

LAYOUT_NCHW, LAYOUT_NHWC = 0, 1
EPI_RELU = 1
EPI_RES_UP2 = 2
EPI_NO_TMA = 4
EPI_STEM_PAIR = 8


def EPI_SIGMOID_FROM(c):
    return ((int(c) + 1) & 0x3ff) << 20
PREC_FP32_SIMT, PREC_BF16X3, PREC_BF16 = 0, 1, 2
DTYPE_F32, DTYPE_BF16, DTYPE_PAIR = 0, 1, 2
LAYOUT_FLAT_PAIR = 2

_ERR = {-1: "bad argument", -2: "unsupported configuration", -3: "workspace too small"}


class UpsnetError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            from . import build as _build  # in-tree nvcc build; raises if nvcc is missing
            _build.build()
        L = C.CDLL(LIB_PATH)
        vp, i, f, d, sz = C.c_void_p, C.c_int, C.c_float, C.c_double, C.c_size_t
        L.upsnet_version.argtypes = [C.POINTER(i)]
        L.upsnet_roi_align_forward.argtypes = [vp, i, i, i, i, i, i, vp, i, i, i, i, f, vp, vp]
        L.upsnet_roi_align_fpn_forward.argtypes = [C.POINTER(vp), C.POINTER(i), C.POINTER(i), C.POINTER(f),
                                                   i, i, i, i, vp, i, i, i, i, vp, vp, vp, vp]
        L.upsnet_nms_workspace_bytes.argtypes = [i, i, C.POINTER(sz)]
        L.upsnet_nms_segmented.argtypes = [vp, vp, i, i, f, vp, vp, vp, sz, vp]
        L.upsnet_nms_host.argtypes = [vp, vp, vp, i, i, f, i]
        L.upsnet_dcn_forward.argtypes = [vp] * 6 + [i] * 16 + [vp]
        L.upsnet_conv2d_forward.argtypes = [vp] * 5 + [i] * 15 + [vp]
        L.upsnet_igemm_packed_weight_bytes.argtypes = [i, i, i, i, C.POINTER(sz)]
        L.upsnet_igemm_pack_weight.argtypes = [vp, i, i, i, i, vp, vp]
        L.upsnet_igemm_forward.argtypes = [vp] * 7 + [i] * 18 + [vp, vp]
        L.upsnet_dcn_packed_weight_bytes.argtypes = [i, i, i, i, C.POINTER(sz)]
        L.upsnet_dcn_pack_weight.argtypes = [vp, i, i, i, i, vp, vp]
        L.upsnet_dcn_pair_forward.argtypes = [vp] * 6 + [i] * 12 + [vp]
        L.upsnet_dcn_set_tile_n.argtypes = [i]
        L.upsnet_tma_set_tile_n.argtypes = [i]
        L.upsnet_panoptic_workspace_bytes.argtypes = [i, i, i, i, C.POINTER(sz)]
        L.upsnet_panoptic_workspace_min_bytes.argtypes = [i, i, i, i, C.POINTER(sz)]
        L.upsnet_panoptic_head.argtypes = [vp, i, i, i, vp, vp, vp, vp, i, vp, i, d, vp, vp, vp, vp, vp, sz, vp]
        L.upsnet_panoptic_head_up4.argtypes = [vp, i, i, i, vp, vp, vp, vp, i, vp, i, d, vp, vp, vp, vp, vp, sz, vp]
        L.upsnet_mask_removal.argtypes = [vp, vp, vp, vp, i, vp, i, i, i, d, vp, vp, vp, vp, sz, vp]
        L.upsnet_rpn_decode.argtypes = [C.POINTER(vp), C.POINTER(vp), C.POINTER(i), C.POINTER(i), C.POINTER(i),
                                        C.POINTER(i), vp, i, i, f, f, vp, vp]
        L.upsnet_maskroi_prepare.argtypes = [vp, vp, vp, vp, i, i, i, f, C.POINTER(f), f, f, vp, vp, vp, vp, vp]
        L.upsnet_maskroi_finish.argtypes = [vp] * 6 + [i] * 4 + [vp] * 5
        L.upsnet_mask_rows.argtypes = [vp, vp, i, vp, vp, i, vp, vp, vp, vp]
        L.upsnet_maxpool2d_nhwc.argtypes = [vp, vp] + [i] * 8 + [vp]
        L.upsnet_upsample_bilinear_nchw.argtypes = [vp, vp, i, i, i, i, vp]
        L.upsnet_rpn_topk_workspace_bytes.argtypes = [i, C.POINTER(sz)]
        L.upsnet_stem_workspace_bytes.argtypes = [i] * 6 + [C.POINTER(sz)]
        L.upsnet_stem_packed_weight_bytes.argtypes = [i, i, C.POINTER(sz)]
        L.upsnet_stem_pack_weight.argtypes = [vp, i, i, i, i, vp, vp]
        L.upsnet_stem_forward.argtypes = [vp] * 4 + [i] * 9 + [vp, sz, vp]
        L.upsnet_rpn_collect.argtypes = [vp] * 5 + [i] * 3 + [vp] * 4
        L.upsnet_rpn_topk.argtypes = [C.POINTER(vp), C.POINTER(i), C.POINTER(i), i, i, i, vp, vp, vp, sz, vp]
        L.upsnet_dcn_im2col.argtypes = [vp, vp, vp] + [i] * 11 + [vp, vp]
        L.upsnet_dcn_col2im.argtypes = [vp, vp, vp] + [i] * 11 + [vp, vp]
        L.upsnet_dcn_col2im_coord.argtypes = [vp, vp, vp, vp] + [i] * 11 + [vp, vp, vp]
        L.upsnet_roi_align_backward.argtypes = [vp, vp] + [i] * 8 + [f, vp, vp]
        L.upsnet_fcn_score_fuse.argtypes = [vp, vp, vp, vp, vp, i, i, i, vp]
        L.upsnet_unified_pan_workspace_bytes.argtypes = [i, C.POINTER(sz)]
        L.upsnet_unified_pan_result.argtypes = [vp, vp, vp, i, vp, i, i, i, i, i, vp, vp, vp, sz, vp]
        L.upsnet_im_post_workspace_bytes.argtypes = [i, i, C.POINTER(sz)]
        L.upsnet_im_post_rle.argtypes = [vp, i, i, vp, vp, i, vp, i, i, vp, i, vp, vp, vp, sz, vp]
        L.upsnet_prep_image.argtypes = [vp, i, i, d, i, i, i, i, C.POINTER(d), vp, vp]
        L.upsnet_label_restore.argtypes = [vp, vp, i, i, i, i, d, i, i, vp, vp, vp]
        L.upsnet_pq_workspace_bytes.argtypes = [C.POINTER(sz)]
        L.upsnet_pq_update.argtypes = [vp, vp, i, i, vp, i, vp, vp, vp, vp, vp, sz, vp]
        L.upsnet_sseg_update.argtypes = [vp, i, i, vp, vp, vp, i, i, i, vp, vp]
        L.upsnet_cocoeval_workspace_bytes.argtypes = [i, i, C.c_longlong, C.POINTER(sz)]
        L.upsnet_cocoeval_image.argtypes = [i, vp, vp, vp, i, vp, vp, i, vp, i, i, vp, i, vp, vp, i, vp, i, vp, i, vp, vp,
                                            vp, vp, sz, vp]
        L.upsnet_cocoeval_accumulate_workspace_bytes.argtypes = [i, C.POINTER(sz)]
        L.upsnet_cocoeval_accumulate.argtypes = [vp, i, vp, vp, i, vp, vp, vp, vp, sz, vp]
        L.upsnet_combined_pan_workspace_bytes.argtypes = [i, i, i, C.POINTER(sz)]
        L.upsnet_combined_pan_result.argtypes = [vp, i, i, i, vp, vp, i, vp, vp, i, vp, i, i, f, f, i, vp, vp, vp, sz, vp]
        L.upsnet_rpn_targets_workspace_bytes.argtypes = [C.c_longlong, i, C.POINTER(sz)]
        L.upsnet_rpn_targets.argtypes = [vp, i, vp, C.POINTER(i), C.POINTER(i), i, i, d, d, d, f, f, i, i, C.c_ulonglong,
                                         vp, vp, vp, vp, vp, vp, sz, vp]
        L.upsnet_proposal_targets_workspace_bytes.argtypes = [i, i, i, C.POINTER(sz)]
        L.upsnet_proposal_targets.argtypes = [vp, i] + [vp] * 5 + [i] + [vp] * 4 + [i, f, i, i, i] + [f] * 7 + \
            [i, i, C.c_ulonglong] + [vp] * 11 + [sz, vp]
        L.upsnet_panoptic_loss_workspace_bytes.argtypes = [i, i, i, C.POINTER(sz)]
        L.upsnet_panoptic_loss_forward.argtypes = [vp, i, i, i, vp, i, i, i, vp, vp, vp, vp, i, i, vp, i, i, f] + \
            [vp] * 6 + [sz, vp]
        L.upsnet_panoptic_loss_backward.argtypes = [vp, i, i, i, vp, i, i, i, vp, vp, i, i, f] + [vp] * 6 + [sz, vp]
        L.upsnet_panoptic_gt.argtypes = [vp, vp, i, i, vp, i, i, i, i, i, vp, vp]
        L.upsnet_draw_keys.argtypes = [C.c_ulonglong, i, i, vp, vp]
        L.upsnet_training_labels.argtypes = [vp, i, i, vp, i, vp, i, vp, vp, i, vp, i, vp, vp, i, vp, i] + [vp] * 4 + \
            [i, i, i, vp, i, vp, vp, i, i, vp, vp]
        _lib = L
    return _lib


EXPORTED_SYMBOLS = [
    "upsnet_version", "upsnet_roi_align_forward", "upsnet_roi_align_fpn_forward",
    "upsnet_nms_workspace_bytes", "upsnet_nms_segmented", "upsnet_nms_host", "upsnet_dcn_forward",
    "upsnet_conv2d_forward", "upsnet_igemm_packed_weight_bytes", "upsnet_igemm_pack_weight",
    "upsnet_igemm_forward", "upsnet_panoptic_workspace_bytes", "upsnet_panoptic_workspace_min_bytes", "upsnet_panoptic_head", "upsnet_panoptic_head_up4", "upsnet_mask_removal",
    "upsnet_rpn_decode", "upsnet_maskroi_prepare", "upsnet_maskroi_finish", "upsnet_mask_rows", "upsnet_maxpool2d_nhwc", "upsnet_upsample_bilinear_nchw", "upsnet_rpn_topk_workspace_bytes", "upsnet_rpn_topk", "upsnet_rpn_collect", "upsnet_stem_workspace_bytes",
    "upsnet_stem_packed_weight_bytes", "upsnet_stem_pack_weight", "upsnet_stem_forward",
    "upsnet_dcn_im2col", "upsnet_dcn_col2im", "upsnet_dcn_col2im_coord", "upsnet_roi_align_backward",
    "upsnet_dcn_packed_weight_bytes", "upsnet_dcn_pack_weight", "upsnet_dcn_pair_forward", "upsnet_dcn_set_tile_n", "upsnet_tma_set_tile_n",
    "upsnet_fcn_score_fuse", "upsnet_unified_pan_workspace_bytes", "upsnet_unified_pan_result", "upsnet_prep_image", "upsnet_im_post_workspace_bytes", "upsnet_im_post_rle",
    "upsnet_label_restore", "upsnet_pq_workspace_bytes", "upsnet_pq_update",
    "upsnet_sseg_update", "upsnet_cocoeval_workspace_bytes", "upsnet_cocoeval_image",
    "upsnet_cocoeval_accumulate_workspace_bytes", "upsnet_cocoeval_accumulate",
    "upsnet_combined_pan_workspace_bytes", "upsnet_combined_pan_result",
    "upsnet_rpn_targets_workspace_bytes", "upsnet_rpn_targets",
    "upsnet_proposal_targets_workspace_bytes", "upsnet_proposal_targets",
    "upsnet_panoptic_loss_workspace_bytes", "upsnet_panoptic_loss_forward", "upsnet_panoptic_loss_backward",
    "upsnet_panoptic_gt", "upsnet_draw_keys", "upsnet_training_labels",
]


def check(rc, what):
    if rc == 0:
        return
    if rc < 0:
        raise UpsnetError("%s: %s (%d)" % (what, _ERR.get(rc, "error"), rc))
    raise UpsnetError("%s: CUDA error %d" % (what, rc))


def stream_ptr(device=None):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(None)


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise UpsnetError("upsnet_b200 ops are CUDA-only (sm_90a); got a %s tensor" % t.device)


def f32c(t):
    """fp32 + contiguous (NCHW), no copy when already so."""
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()
