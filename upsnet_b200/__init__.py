"""upsnet_b200 -- H100-native (sm_90a) implementation of the UPSNet per-image inference hot path
behind the reference's own operator API.  All compute lives in libupsnet_b200.so (C ABI:
include/upsnet_b200.h); this package is the thin PyTorch-facing host layer."""
from .operators import (DeformConv, DeformConvWithOffset, ModDeformConv, ModDeformConvWithOffsetMask,  # noqa: F401
                        ModulatedDeformConv, RoIAlign, ROIAlign, RoIAlignFunction, FPNRoIAlign, PanopticHead,
                        MaskRemoval, SegTerm, MaskTerm, MaskMatching,
                        conv2d, linear, deform_conv, roi_align, fpn_roi_align, nms, nms_segmented, gpu_nms,
                        gpu_nms_wrapper, panoptic_fuse, set_precision, unified_pan_result, prep_image, im_post, im_post_rle,
                        label_restore, combined_pan_result, get_combined_pan_result)

from .pipeline import PipelinedEngine  # noqa: F401,E402
from .evaluation import PanopticQuality, SegmentationIoU, DetectionAP  # noqa: F401,E402
from .training import (Conv2dFunction, ConvTranspose2x2Function, FlatBucketAllReduce, LRSchedule,  # noqa: F401,E402
                       FcnRoiLoss, MaskRCNNLoss, PanopticLabels, PanopticLoss, RPNLoss, SemanticLoss, SGD,
                       TrainingSample)

__all__ = ["PipelinedEngine", "DeformConv", "DeformConvWithOffset", "ModDeformConv", "ModDeformConvWithOffsetMask",
           "ModulatedDeformConv", "RoIAlign", "ROIAlign", "RoIAlignFunction", "FPNRoIAlign", "PanopticHead",
           "MaskRemoval", "SegTerm", "MaskTerm", "MaskMatching",
           "conv2d", "linear", "deform_conv", "roi_align", "fpn_roi_align", "nms", "nms_segmented", "gpu_nms",
           "gpu_nms_wrapper", "panoptic_fuse", "set_precision", "unified_pan_result", "prep_image", "im_post", "im_post_rle",
           "label_restore", "combined_pan_result", "get_combined_pan_result", "PanopticQuality", "SegmentationIoU", "DetectionAP",
           "PanopticLoss", "PanopticLabels", "TrainingSample", "SemanticLoss", "FcnRoiLoss", "RPNLoss", "MaskRCNNLoss", "SGD", "LRSchedule",
           "FlatBucketAllReduce", "Conv2dFunction", "ConvTranspose2x2Function"]
