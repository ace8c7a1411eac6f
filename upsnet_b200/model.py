"""resnet_upsnet inference engine: the host-side mirror of upsnet/models/{resnet,fpn,rpn,rcnn,fcn,
resnet_upsnet}.py running on the sm_90a C ABI.

* Same module tree / parameter names as the reference, so its checkpoints load with
  load_state_dict (e.g. resnet_backbone.res3.layers.0.conv2_offset.weight,
  fcn_head.fcn_subnet.conv.0.0.conv_offset.weight; SURVEY.md section 5 "Checkpoint / resume").
* forward(data, label=None) -> the reference's result dict (models/resnet_upsnet.py:209-247):
  cls_probs, pred_boxes, mask_probs, fcn_outputs, cls_inds, panoptic_cls_inds,
  panoptic_cls_probs, panoptic_outputs.
* Frozen BatchNorm (models/resnet.py:69-78: always eval, requires_grad False) is folded into the
  preceding convolution once (prepare()); bias/ReLU/residual live in the conv epilogue.
* forward(data, label) -> the reference's training outputs (models/resnet_upsnet.py:88-195; one image): rpn_cls_loss,
  rpn_bbox_loss, cls_loss, bbox_loss, mask_loss, fcn_loss, panoptic_loss, rcnn_accuracy, panoptic_accuracy, each
  float32 [1] on the device, plus fcn_roi_loss (float32 [], as the reference returns it) when train.fcn_with_roi_loss
  is set (every COCO configuration, which also sets network.fpn_with_gap: FPN's context vector folded into the P5
  lateral conv's bias).
  An eager autograd path separate from the static engine: every module has forward_train(..., prec) next to its
  forward, built from training.conv2d / linear / conv_transpose2x2 with BN folded per call, the DCN / ROIAlign backward Functions and, in the semantic head, the level sum through
  FcnScoreFuseFunction; _forward_train composes them with the targets and the device losses (FcnRoiLoss for the
  semantic head's ROI loss, which samples fcn_score instead of the 512-channel concat).
  get_params_lr() gives the reference's 13 parameter groups for upsnet_b200.SGD.
"""
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib, training
from . import operators as ops
from .detection import MaskROI, ProposalGenerator, StaticMaskROI, StaticProposalGenerator
from .operators import DeformConv, DeformConvWithOffset


class UPSNetConfig:
    """The hot-path knobs of upsnet/config/config.py + experiments/*.yaml."""

    def __init__(self, **kw):
        self.num_classes = 9              # dataset.num_classes (Cityscapes: 8 things + bg)
        self.num_seg_classes = 19         # dataset.num_seg_classes
        self.backbone_with_dconv = 100    # network.backbone_with_dconv (3 => DCN in res3..res5)
        self.backbone_with_dilation = False
        self.backbone_with_dpyramid = False
        self.backbone_freeze_at = 2       # network.backbone_freeze_at: conv1 and res2..res<freeze_at> get no gradient
        self.backbone_fix_bn = True       # network.backbone_fix_bn: BatchNorm frozen (eval statistics, no gradient)
        self.fpn_feature_dim = 256
        self.fpn_with_gap = False
        self.fcn_num_layers = 2
        self.num_anchors = 3
        self.anchor_scales = (8,)
        self.anchor_ratios = (0.5, 1, 2)
        self.rpn_feat_stride = (4, 8, 16, 32, 64)
        self.mask_size = 28
        self.bbox_reg_weights = (10., 10., 5., 5.)
        self.rpn_pre_nms_top_n = 1000
        self.rpn_post_nms_top_n = 1000
        self.rpn_nms_thresh = 0.7
        self.rpn_min_size = 0
        self.nms_thresh = 0.5
        self.max_det = 100
        self.score_thresh = 0.05
        self.panoptic_score_thresh = 0.6
        self.panoptic_box_keep_fraction = 0.7   # < 1 => enable_void (resnet_upsnet.py:66-67)
        # training forward (config.train.*): proposals, sampling, loss normalisers
        self.train_rpn_pre_nms_top_n = 2000
        self.train_rpn_post_nms_top_n = 2000
        self.train_rpn_nms_thresh = 0.7
        self.train_rpn_min_size = 0
        self.batch_rois = 512
        self.rpn_batch_size = 256
        self.fg_fraction = 0.25
        self.fcn_with_roi_loss = False
        # network.{fpn,rpn,rcnn,fcn}_with_norm: 'none' or 'group_norm' (nn.GroupNorm(32, C) after each conv of the head);
        # 'batch_norm' needs the reference's absent distbatchnorm module and is refused by resnet_upsnet
        self.fpn_with_norm = "none"
        self.rpn_with_norm = "none"
        self.rcnn_with_norm = "none"
        self.fcn_with_norm = "none"
        # network.fpn_upsample_method: how the FPN's top-down path up-samples the coarser level, 'nearest' or 'bilinear'
        # (F.interpolate(scale_factor=2, align_corners=False), models/fpn.py:27-35)
        self.fpn_upsample_method = "nearest"
        for k, v in kw.items():
            if not hasattr(self, k):
                raise AttributeError(k)
            setattr(self, k, v)

    @classmethod
    def from_reference_config(cls, config):
        """Build from the reference's global `config` (upsnet/config/config.py + an experiment yaml merged by
        update_config): the fields resnet_upsnet.__init__ reads (models/resnet_upsnet.py:42-71, resnet.py:314-340)."""
        def get(sec, key, default):
            d = config.get(sec, {}) if hasattr(config, "get") else getattr(config, sec, {})
            try:
                return d[key]
            except (KeyError, TypeError):
                return getattr(d, key, default)
        return cls(num_classes=int(get("dataset", "num_classes", 9)), num_seg_classes=int(get("dataset", "num_seg_classes", 19)),
                   backbone_with_dconv=int(get("network", "backbone_with_dconv", 100)),
                   backbone_with_dilation=bool(get("network", "backbone_with_dilation", False)),
                   backbone_with_dpyramid=bool(get("network", "backbone_with_dpyramid", False)),
                   backbone_freeze_at=int(get("network", "backbone_freeze_at", 2)),
                   backbone_fix_bn=bool(get("network", "backbone_fix_bn", True)),
                   fpn_feature_dim=int(get("network", "fpn_feature_dim", 256)), fpn_with_gap=bool(get("network", "fpn_with_gap", False)),
                   fcn_num_layers=int(get("network", "fcn_num_layers", 3)), num_anchors=int(get("network", "num_anchors", 3)),
                   anchor_scales=tuple(get("network", "anchor_scales", (8,))), anchor_ratios=tuple(get("network", "anchor_ratios", (0.5, 1, 2))),
                   rpn_feat_stride=tuple(get("network", "rpn_feat_stride", (4, 8, 16, 32, 64))), mask_size=int(get("network", "mask_size", 28)),
                   bbox_reg_weights=tuple(get("network", "bbox_reg_weights", (10., 10., 5., 5.))),
                   rpn_pre_nms_top_n=int(get("test", "rpn_pre_nms_top_n", 1000)), rpn_post_nms_top_n=int(get("test", "rpn_post_nms_top_n", 1000)),
                   rpn_nms_thresh=float(get("test", "rpn_nms_thresh", 0.7)), rpn_min_size=int(get("test", "rpn_min_size", 0)),
                   nms_thresh=float(get("test", "nms_thresh", 0.5)), max_det=int(get("test", "max_det", 100)),
                   score_thresh=float(get("test", "score_thresh", 0.05)), panoptic_score_thresh=float(get("test", "panoptic_score_thresh", 0.6)),
                   panoptic_box_keep_fraction=float(get("train", "panoptic_box_keep_fraction", 0.7)),
                   train_rpn_pre_nms_top_n=int(get("train", "rpn_pre_nms_top_n", 2000)),
                   train_rpn_post_nms_top_n=int(get("train", "rpn_post_nms_top_n", 2000)),
                   train_rpn_nms_thresh=float(get("train", "rpn_nms_thresh", 0.7)),
                   train_rpn_min_size=int(get("train", "rpn_min_size", 0)),
                   batch_rois=int(get("train", "batch_rois", 512)), rpn_batch_size=int(get("train", "rpn_batch_size", 256)),
                   fg_fraction=float(get("train", "fg_fraction", 0.25)),
                   fcn_with_roi_loss=bool(get("train", "fcn_with_roi_loss", False)),
                   fpn_upsample_method=str(get("network", "fpn_upsample_method", "nearest")),
                   **{k: str(get("network", k, "none")) for k in NORM_KEYS})

    @classmethod
    def cityscapes_r50(cls):      # experiments/upsnet_resnet50_cityscapes_16gpu.yaml
        return cls()

    @classmethod
    def coco_r50(cls):            # experiments/upsnet_resnet50_coco_{4,8,16}gpu.yaml
        return cls(num_classes=81, num_seg_classes=133, fpn_with_gap=True, fcn_num_layers=3, fcn_with_roi_loss=True)

    @classmethod
    def coco_r101_dcn(cls):       # experiments/upsnet_resnet101_dcn_coco_3x_16gpu.yaml
        return cls(num_classes=81, num_seg_classes=133, backbone_with_dconv=3, fpn_with_gap=True,
                   fcn_num_layers=3, fcn_with_roi_loss=True)


NORM_KEYS = ("fpn_with_norm", "rpn_with_norm", "rcnn_with_norm", "fcn_with_norm")


def _check_norms(cfg):
    """The reference builds nn.GroupNorm(32, C) for 'group_norm'; its 'batch_norm' is a BatchNorm2d imported only from
    the absent distbatchnorm module (models/fpn.py:22-23), so it raises NameError there and UpsnetError here.
    rpn_with_norm is read but unused: models/resnet_upsnet.py:52 builds the RPN without passing it."""
    for k in NORM_KEYS:
        v = getattr(cfg, k)
        if v not in ("none", "group_norm", "batch_norm"):
            raise _lib.UpsnetError("network.%s: %r is not one of 'none', 'group_norm', 'batch_norm'" % (k, v))
        if v == "batch_norm" and k != "rpn_with_norm":
            raise _lib.UpsnetError("network.%s = 'batch_norm' is not built: the reference's BatchNorm2d comes from its "
                                   "absent distbatchnorm module (SyncBN); use 'group_norm' or 'none'" % k)


def _check_fpn_upsample(cfg):
    """The reference's FPN asserts upsample_method in ['nearest', 'bilinear'] (models/fpn.py:31)."""
    if cfg.fpn_upsample_method not in ("nearest", "bilinear"):
        raise _lib.UpsnetError("network.fpn_upsample_method: %r is not one of 'nearest', 'bilinear'"
                               % (cfg.fpn_upsample_method,))


def _gn_conv(cin, cout, k, padding=0):
    """conv (no bias) + nn.GroupNorm(32, cout): the reference's normed conv (models/fpn.py:47-54)."""
    return nn.Sequential(nn.Conv2d(cin, cout, k, padding=padding, bias=False), nn.GroupNorm(32, cout))


def _fold_bn(conv_w, bn):
    """Frozen BatchNorm folded into the preceding conv: (conv_w * scale, shift), differentiable in conv_w only.
    prepare() detaches the result; forward_train keeps it, so autograd carries d weight back to the unfolded weight."""
    with torch.no_grad():
        scale = bn.weight / torch.sqrt(bn.running_var + bn.eps)
        shift = (bn.bias - bn.running_mean * scale).contiguous()
    return (conv_w * scale.view(-1, 1, 1, 1)).contiguous(), shift


# ---------------------------------------------------------------------------------------------
# backbone (models/resnet.py)
# ---------------------------------------------------------------------------------------------
class Bottleneck(nn.Module):
    """models/resnet.py:53-100 (and :102-153 when deformable): 1x1(stride) -> 3x3 -> 1x1, +res."""

    def __init__(self, inplanes, planes, stride=1, dilation=1, downsample=None, deformable=False):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 1, stride=stride, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.deformable = deformable
        if deformable:
            self.conv2_offset = nn.Conv2d(planes, 18, 3, 1, 1)
            self.conv2_offset.weight.data.zero_()
            self.conv2_offset.bias.data.zero_()
            self.conv2 = DeformConv(planes, planes, 3, stride=1, padding=dilation, dilation=dilation, bias=False)
        else:
            self.conv2 = nn.Conv2d(planes, planes, 3, 1, dilation, dilation, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.downsample = downsample
        self.stride, self.dilation = stride, dilation
        self._f = None

    def prepare(self):
        f = {}
        f["w1"], f["b1"] = _fold_bn(self.conv1.weight, self.bn1)
        f["w2"], f["b2"] = _fold_bn(self.conv2.weight, self.bn2)
        f["w3"], f["b3"] = _fold_bn(self.conv3.weight, self.bn3)
        if self.downsample is not None:
            f["wd"], f["bd"] = _fold_bn(self.downsample[0].weight, self.downsample[1])
        self._f = {k: v.detach() for k, v in f.items()}

    def forward(self, x):
        f = self._f
        out = ops.conv2d(x, f["w1"], f["b1"], stride=self.stride, relu=True)
        if self.deformable:
            offset = ops.conv2d(out, self.conv2_offset.weight, self.conv2_offset.bias, 1, 1, 1, out_format="nchw")
            out = ops.deform_conv(out, offset, f["w2"], f["b2"], 1, self.dilation, self.dilation, relu=True)
        else:
            out = ops.conv2d(out, f["w2"], f["b2"], 1, self.dilation, self.dilation, relu=True)
        residual = x if self.downsample is None else ops.conv2d(x, f["wd"], f["bd"], stride=self.stride)
        return ops.conv2d(out, f["w3"], f["b3"], residual=residual, relu=True)

    def forward_train(self, x, prec):
        """forward with device gradients: the dense convs through training.conv2d with BN folded per call, the
        deformable 3x3 through OffsetConvFunction / DeformConvFunction."""
        w1, b1 = _fold_bn(self.conv1.weight, self.bn1)
        out = training.conv2d(x, w1, b1, stride=self.stride, relu=True, precision=prec)
        w2, b2 = _fold_bn(self.conv2.weight, self.bn2)
        if self.deformable:
            offset = training.OffsetConvFunction.apply(out, self.conv2_offset.weight, self.conv2_offset.bias)
            out = F.relu(training.DeformConvFunction.apply(out, offset, w2, b2, 1, self.dilation, self.dilation))
        else:
            out = training.conv2d(out, w2, b2, 1, self.dilation, self.dilation, relu=True, precision=prec)
        residual = x
        if self.downsample is not None:
            wd, bd = _fold_bn(self.downsample[0].weight, self.downsample[1])
            residual = training.conv2d(x, wd, bd, stride=self.stride, precision=prec)
        w3, b3 = _fold_bn(self.conv3.weight, self.bn3)
        return training.conv2d(out, w3, b3, residual=residual, relu=True, precision=prec)


class Stem(nn.Module):
    """models/resnet.py:155-175 `conv1`: 7x7/2 conv + BN + ReLU + 3x3/2 max-pool."""

    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 64, 7, 2, 3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self._f = None

    def prepare(self):
        w, b = _fold_bn(self.conv1.weight, self.bn1)
        self._f = (w.detach(), b.detach())

    def forward(self, x):
        stream = ops._stream()
        if x.is_cuda and stream != "f32":       # bf16 / pair stream: the TMA-fed stem
            x = ops.stem_conv(x, self._f[0], self._f[1], 3, relu=True, pair=stream == "pair")
        else:       # fp32 stream, and CPU tensors (oracle.cpu_model.cpu_ops swaps in CPU versions of ops.conv2d & co.)
            x = ops.conv2d(x, self._f[0], self._f[1], stride=2, padding=3, relu=True)
        return ops.max_pool2d(x, 3, 2, 1)


class ResBlock(nn.Module):
    """models/resnet.py:177-207 res_block; parameters live under `.layers.<i>`."""

    def __init__(self, planes, blocks, stride=1, dilation=1, deformable=False, with_dpyramid=False):
        super().__init__()
        inplanes = planes * 2 if planes != 64 else planes
        downsample = None
        if stride != 1 or inplanes != planes * 4:
            downsample = nn.Sequential(nn.Conv2d(inplanes, planes * 4, 1, stride=stride, bias=False),
                                       nn.BatchNorm2d(planes * 4))
        layers = [Bottleneck(inplanes, planes, stride, dilation, downsample, deformable)]
        for _ in range(1, blocks - 1):
            layers.append(Bottleneck(planes * 4, planes, dilation=dilation, deformable=deformable))
        layers.append(Bottleneck(planes * 4, planes, dilation=dilation, deformable=deformable or with_dpyramid))
        self.layers = nn.Sequential(*layers)

    def forward(self, x):
        return self.layers(x)


class ResNetBackbone(nn.Module):
    """models/resnet.py:314-356."""

    def __init__(self, blocks, cfg):
        super().__init__()
        d = cfg.backbone_with_dconv
        self.conv1 = Stem()
        self.res2 = ResBlock(64, blocks[0])
        self.res3 = ResBlock(128, blocks[1], 2, deformable=d <= 3, with_dpyramid=cfg.backbone_with_dpyramid)
        self.res4 = ResBlock(256, blocks[2], 2, deformable=d <= 4, with_dpyramid=cfg.backbone_with_dpyramid)
        s5, d5 = (1, 2) if cfg.backbone_with_dilation else (2, 1)
        self.res5 = ResBlock(512, blocks[3], s5, d5, deformable=d <= 5)

    def forward(self, x):
        c1 = self.conv1(x)
        r2 = self.res2(c1)
        r3 = self.res3(r2)
        r4 = self.res4(r3)
        return r2, r3, r4, self.res5(r4)

    def forward_train(self, x, prec):
        """r2 .. r5 of the training forward: the frozen stem and res2 (backbone_freeze_at = 2) on the inference path
        under no_grad, folded afresh, then res3 - res5 with device gradients."""
        with torch.no_grad():
            for m in [self.conv1] + list(self.res2.layers):
                m.prepare()
            r = ops.as_float(self.res2(self.conv1(x))).float()
        out = [r]
        for stage in (self.res3, self.res4, self.res5):
            for blk in stage.layers:
                r = blk.forward_train(r, prec)
            out.append(r)
        return tuple(out)


# ---------------------------------------------------------------------------------------------
# FPN / RPN / heads (models/fpn.py, rpn.py, rcnn.py, fcn.py)
# ---------------------------------------------------------------------------------------------
class FPN(nn.Module):
    """models/fpn.py:25-104 (with_norm 'none' or 'group_norm', upsample_method 'nearest' or 'bilinear', P6 = stride-2
    subsample of P5).  The up-sampling method has no parameters: both build the same module tree."""

    def __init__(self, feature_dim, with_gap, with_norm="none", upsample_method="nearest"):
        super().__init__()
        self.feature_dim = feature_dim
        self.gn = with_norm == "group_norm"
        self.upsample_method = upsample_method
        if with_gap:
            self.fpn_gap = nn.Linear(2048, feature_dim)
        for name, cin in (("fpn_p5_1x1", 2048), ("fpn_p4_1x1", 1024), ("fpn_p3_1x1", 512), ("fpn_p2_1x1", 256)):
            setattr(self, name, _gn_conv(cin, feature_dim, 1) if self.gn else nn.Conv2d(cin, feature_dim, 1))
        for name in ("fpn_p5", "fpn_p4", "fpn_p3", "fpn_p2"):
            setattr(self, name, _gn_conv(feature_dim, feature_dim, 3, 1) if self.gn else
                    nn.Conv2d(feature_dim, feature_dim, 3, padding=1))
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_uniform_(m.weight.data, a=1)
                if m.bias is not None:
                    m.bias.data.zero_()

    def forward(self, res2, res3, res4, res5):
        """Each lateral 1x1 ends in an epilogue that adds the 2x-upsampled coarser level: with 'none' the conv's, after
        its bias; with 'group_norm' the GN apply's, after a conv without bias.  With 'nearest' both epilogues read the
        coarser level directly, so no upsampled tensor is written; with 'bilinear' the GN apply reads its four bilinear
        taps, and with 'none' the up-sampling kernel writes the upsampled map, which the conv adds as a plain residual.
        The context vector fpn_gap(GAP(res5)) is the P5 lateral's GN shift, or with 'none' added to that conv's output;
        either way it is in P5's lateral before that is up-sampled (models/fpn.py:84-88)."""
        bilinear = self.upsample_method == "bilinear"

        def step(name, x, padding=0, residual=None, shift=None):
            up = {"residual": residual, "residual_up2": residual is not None}
            if not self.gn:
                m = getattr(self, name)
                if bilinear and residual is not None:
                    up = {"residual": ops.upsample2_bilinear(residual)}
                return ops.conv2d(x, m.weight, m.bias, padding=padding, **up)
            conv, gn = getattr(self, name)
            t = ops.conv2d(x, conv.weight, None, padding=padding)
            return ops.group_norm(t, gn.weight, gn.bias, gn.num_groups, gn.eps, shift=shift,
                                  upsample=self.upsample_method, **up)

        def gap():          # models/fpn.py:84-86, float32 [N, C]; launched where each norm consumes it
            return ops.linear(res5.float().mean(dim=(2, 3)), self.fpn_gap.weight, self.fpn_gap.bias, out_dtype=torch.float32)
        with_gap = hasattr(self, "fpn_gap")
        p5_1x1 = step("fpn_p5_1x1", res5, shift=gap() if with_gap and self.gn else None)
        if with_gap and not self.gn:
            g = gap().view(-1, self.feature_dim, 1, 1)
            if isinstance(p5_1x1, ops.Pair):
                p5_1x1 = ops.Pair.from_float(p5_1x1.float() + g)
            else:
                p5_1x1 = p5_1x1 + g.to(p5_1x1.dtype)
        p4_plus = step("fpn_p4_1x1", res4, residual=p5_1x1)
        p3_plus = step("fpn_p3_1x1", res3, residual=p4_plus)
        p2_plus = step("fpn_p2_1x1", res2, residual=p3_plus)
        p5 = step("fpn_p5", p5_1x1, padding=1)
        p4 = step("fpn_p4", p4_plus, padding=1)
        p3 = step("fpn_p3", p3_plus, padding=1)
        p2 = step("fpn_p2", p2_plus, padding=1)
        p6 = ops.subsample2(p5)                                         # MaxPool2d(kernel 1, stride 2)
        return p2, p3, p4, p5, p6

    def forward_train(self, res2, res3, res4, res5, prec):
        """forward with device gradients: training.conv2d, then with group_norm training.group_norm, with the same fused
        top-down add ('bilinear' with 'none': training.upsample2_bilinear, whose backward is the adjoint kernel, then
        the plain residual).  The context vector fpn_gap(GAP(res5)) (models/fpn.py:84-86, added to every P5 lateral
        pixel) is, with 'none', folded into the bias of the P5 lateral conv, so that conv's d bias carries the gradient
        to both biases, fpn_gap and res5; with 'group_norm' it is the GN apply's shift, whose gradient the GN backward
        returns."""
        bilinear = self.upsample_method == "bilinear"

        def step(name, x, padding=0, residual=None, shift=None):
            if not self.gn:
                m = getattr(self, name)
                bias = m.bias if shift is None else m.bias + shift.reshape(self.feature_dim)
                if bilinear and residual is not None:
                    return training.conv2d(x, m.weight, bias, padding=padding,
                                           residual=training.upsample2_bilinear(residual), precision=prec)
                return training.conv2d(x, m.weight, bias, padding=padding, residual=residual,
                                       residual_up2=residual is not None, precision=prec)
            conv, gn = getattr(self, name)
            t = training.conv2d(x, conv.weight, None, padding=padding, precision=prec)
            return training.group_norm(t, gn.weight, gn.bias, gn.num_groups, gn.eps, residual=residual, shift=shift,
                                       upsample=self.upsample_method)

        gap = None
        if hasattr(self, "fpn_gap"):        # one image: the context vector is one row
            gap = training.linear(res5.mean((2, 3)), self.fpn_gap.weight, self.fpn_gap.bias, precision=prec)
        p5_1x1 = step("fpn_p5_1x1", res5, shift=gap)
        p4_plus = step("fpn_p4_1x1", res4, residual=p5_1x1)
        p3_plus = step("fpn_p3_1x1", res3, residual=p4_plus)
        p2_plus = step("fpn_p2_1x1", res2, residual=p3_plus)
        p2 = step("fpn_p2", p2_plus, padding=1)
        p3 = step("fpn_p3", p3_plus, padding=1)
        p4 = step("fpn_p4", p4_plus, padding=1)
        p5 = step("fpn_p5", p5_1x1, padding=1)
        return p2, p3, p4, p5, p5[:, :, ::2, ::2]


class RPN(nn.Module):
    """models/rpn.py:26-57."""

    def __init__(self, num_anchors, input_dim):
        super().__init__()
        self.num_anchors = num_anchors
        self.conv_proposal = nn.Sequential(nn.Conv2d(input_dim, input_dim, 3, padding=1), nn.ReLU(inplace=True))
        self.cls_score = nn.Conv2d(input_dim, num_anchors, 1)
        self.bbox_pred = nn.Conv2d(input_dim, num_anchors * 4, 1)
        for m in (self.conv_proposal[0], self.cls_score, self.bbox_pred):
            nn.init.normal_(m.weight.data, 0, 0.01)
            m.bias.data.zero_()
        self._f = None

    def prepare(self):
        # the two 1x1 heads share their input: one GEMM with Cout = A + 4A + A -- the last A rows repeat cls_score and get
        # the sigmoid in the epilogue (models/rpn.py:55), so logits, deltas and probabilities leave one launch
        self._f = (torch.cat([self.cls_score.weight, self.bbox_pred.weight, self.cls_score.weight]).detach().contiguous(),
                   torch.cat([self.cls_score.bias, self.bbox_pred.bias, self.cls_score.bias]).detach().contiguous())

    def forward(self, x):
        c = self.conv_proposal[0]
        t = ops.conv2d(x, c.weight, c.bias, padding=1, relu=True)
        A = self.num_anchors
        both = ops.conv2d(t, self._f[0], self._f[1], out_format="nchw", sigmoid_from=5 * A).float()
        return both[:, :A], both[:, A:5 * A], both[:, 5 * A:]

    def forward_train(self, x, prec):
        """(cls_score, bbox_pred) logits of one level with device gradients: the shared 3x3 + ReLU, then the two 1x1
        heads as separate convs."""
        c = self.conv_proposal[0]
        t = training.conv2d(x, c.weight, c.bias, padding=1, relu=True, precision=prec)
        return (training.conv2d(t, self.cls_score.weight, self.cls_score.bias, precision=prec),
                training.conv2d(t, self.bbox_pred.weight, self.bbox_pred.bias, precision=prec))


class RCNN(nn.Module):
    """models/rcnn.py:89-146."""

    def __init__(self, num_classes, num_reg_classes, pool_size=7, dim_in=256, dim_hidden=1024, with_norm="none"):
        super().__init__()
        self.pool_size = pool_size
        self.roi_pooling = ops.FPNRoIAlign(pool_size, pool_size, [1.0 / 4, 1.0 / 8, 1.0 / 16, 1.0 / 32])
        self.gn = with_norm == "group_norm"
        if self.gn:     # models/rcnn.py:102: Linear, View(-1, C, 1, 1), GroupNorm, View(-1, C), ReLU
            self.fc6 = nn.Sequential(nn.Linear(pool_size ** 2 * dim_in, dim_hidden), nn.Unflatten(1, (dim_hidden, 1, 1)),
                                     nn.GroupNorm(32, dim_hidden), nn.Flatten(), nn.ReLU(inplace=True))
        else:
            self.fc6 = nn.Sequential(nn.Linear(pool_size ** 2 * dim_in, dim_hidden), nn.ReLU(inplace=True))
        self.fc7 = nn.Sequential(nn.Linear(dim_hidden, dim_hidden), nn.ReLU(inplace=True))
        self.cls_score = nn.Linear(dim_hidden, num_classes)
        self.bbox_pred = nn.Linear(dim_hidden, num_reg_classes * 4)
        for m in (self.fc6[0], self.fc7[0]):
            nn.init.kaiming_uniform_(m.weight.data, a=1)
            m.bias.data.fill_(0)
        nn.init.normal_(self.cls_score.weight.data, 0, 0.01)
        self.cls_score.bias.data.fill_(0)
        nn.init.normal_(self.bbox_pred.weight.data, 0, 0.001)
        self.bbox_pred.bias.data.fill_(0)
        self.num_classes = num_classes
        self._f = None

    def prepare(self):
        self._f = (torch.cat([self.cls_score.weight, self.bbox_pred.weight]).detach().contiguous(),
                   torch.cat([self.cls_score.bias, self.bbox_pred.bias]).detach().contiguous())
        # fc6 consumes the flattened (c, ph, pw) roi feature; the engine's ROIAlign writes (ph, pw, c) (NHWC), so
        # keep a column-permuted copy of the weight instead of transposing 1000x12544 activations every image
        w6 = self.fc6[0].weight.detach()
        ps = self.pool_size
        self._w6_nhwc = w6.view(w6.shape[0], -1, ps, ps).permute(0, 2, 3, 1).reshape(w6.shape[0], -1).contiguous()

    def forward(self, feat, rois):
        if isinstance(feat[0], ops.Pair):
            # hi/lo pair stream: ROIAlign writes the flattened (ph, pw, c) feature as one pair 'pixel' per roi
            ps = self.pool_size
            x = ops.fpn_roi_align(list(feat), rois, ps, ps, self.roi_pooling.spatial_scale, layout="flat_pair")
            w6 = self._w6_nhwc
        else:
            pool = self.roi_pooling(feat, rois)
            nhwc = pool.permute(0, 2, 3, 1)
            if self._f is not None and nhwc.is_contiguous() and not pool.is_contiguous():
                x, w6 = nhwc.reshape(pool.size(0), -1), self._w6_nhwc
            else:
                x, w6 = pool.reshape(pool.size(0), -1), self.fc6[0].weight
        fc6 = ops.linear(x, w6, self.fc6[0].bias, relu=not self.gn)
        if self.gn:
            gn = self.fc6[2]
            fc6 = ops.group_norm_rows(fc6, gn.weight, gn.bias, gn.num_groups, gn.eps, relu=True)
        fc7 = ops.linear(fc6, self.fc7[0].weight, self.fc7[0].bias, relu=True)
        both = ops.linear(fc7, self._f[0], self._f[1], out_dtype=torch.float32).float()
        return {"cls_score": both[:, :self.num_classes].contiguous(),
                "bbox_pred": both[:, self.num_classes:].contiguous(), "fc_feat": fc7}

    def forward_train(self, feat, rois, prec):
        """(cls_score, bbox_pred) with device gradients: FPNRoIAlignFunction on the fp32 levels, then fc6, fc7 and the
        two heads as separate training.linear calls."""
        ps = self.pool_size
        pool = training.FPNRoIAlignFunction.apply(rois, ps, ps, self.roi_pooling.spatial_scale, 2, *feat)
        fc6 = training.linear(pool.reshape(pool.shape[0], -1), self.fc6[0].weight, self.fc6[0].bias, relu=not self.gn,
                              precision=prec)
        if self.gn:
            gn = self.fc6[2]
            fc6 = training.group_norm(fc6, gn.weight, gn.bias, gn.num_groups, gn.eps, relu=True)
        fc7 = training.linear(fc6, self.fc7[0].weight, self.fc7[0].bias, relu=True, precision=prec)
        return (training.linear(fc7, self.cls_score.weight, self.cls_score.bias, precision=prec),
                training.linear(fc7, self.bbox_pred.weight, self.bbox_pred.bias, precision=prec))


class MaskBranch(nn.Module):
    """models/rcnn.py:34-87: ROIAlign 14x14 -> 4 x (3x3 + ReLU) -> deconv 2x2/2 + ReLU -> 1x1."""

    def __init__(self, num_classes, mask_size=28, dim_in=256, dim_hidden=256, with_norm="none"):
        super().__init__()
        self.roi_pooling = ops.FPNRoIAlign(mask_size // 2, mask_size // 2, [1.0 / 4, 1.0 / 8, 1.0 / 16, 1.0 / 32])
        self.gn = with_norm == "group_norm"
        for i, cin in enumerate((dim_in, dim_hidden, dim_hidden, dim_hidden), start=1):
            layers = [nn.Conv2d(cin, dim_hidden, 3, 1, 1, bias=False), nn.GroupNorm(32, dim_hidden)] if self.gn else \
                [nn.Conv2d(cin, dim_hidden, 3, 1, 1)]
            setattr(self, "mask_conv%d" % i, nn.Sequential(*layers, nn.ReLU(inplace=True)))
        self.mask_deconv1 = nn.Sequential(nn.ConvTranspose2d(dim_hidden, dim_hidden, 2, 2, 0), nn.ReLU(inplace=True))
        self.mask_score = nn.Conv2d(dim_hidden, num_classes, 1)
        for m in self.modules():
            if isinstance(m, (nn.Conv2d, nn.ConvTranspose2d)):
                nn.init.kaiming_normal_(m.weight.data, mode="fan_in")
                if m.bias is not None:
                    m.bias.data.zero_()
        self._f = None

    def prepare(self):
        # ConvTranspose2d(k=2,s=2): out[n,co,2i+a,2j+b] = sum_ci x[n,ci,i,j] W[ci,co,a,b] + bias[co]
        # == 1x1 conv to 4*Cout channels ordered (a,b,co) followed by a pixel shuffle.
        w = self.mask_deconv1[0].weight                      # [Cin, Cout, 2, 2]
        cin, cout = w.shape[0], w.shape[1]
        w1 = w.permute(2, 3, 1, 0).reshape(4 * cout, cin, 1, 1).detach().contiguous()
        b1 = self.mask_deconv1[0].bias.repeat(4).detach().contiguous()
        self._f = (w1, b1, cout)

    def forward(self, feat, rois, n_dev=None):
        """n_dev (static engine): int32 device count of the rois that are needed -- the pair-stream ROIAlign and the
        tensor-core convs skip the rest, whose logits are then unspecified."""
        bound = {} if n_dev is None else {"n_dev": n_dev}     # (the CPU stand-ins of the ops take no count)
        if n_dev is None or not isinstance(feat[0], ops.Pair):
            x = self.roi_pooling(feat, rois)
        else:
            r = self.roi_pooling
            x = ops.fpn_roi_align(list(feat), rois, r.pooled_height, r.pooled_width, r.spatial_scale, layout="auto", **bound)
        for i in range(1, 5):
            c = getattr(self, "mask_conv%d" % i)
            x = ops.conv2d(x, c[0].weight, c[0].bias, padding=1, relu=not self.gn, **bound)
            if self.gn:
                x = ops.group_norm_rows(x, c[1].weight, c[1].bias, c[1].num_groups, c[1].eps, relu=True, n_dev=n_dev)
        w1, b1, cout = self._f
        if isinstance(x, ops.Pair):
            # pair stream: the deconv-as-1x1 conv writes its four (a, b) groups as [hi Cout][lo Cout] each, i.e. directly
            # as the Pair of 4w 'pixels' per row that mask_score (1x1) then scores -- same commutation as below
            yv = ops.conv2d(x, w1, b1, relu=True, pair_group=cout, **bound)                     # Pair [n, Cout, h, 4w]
            n, _, h, w4 = yv.shape
            w = w4 // 4
        else:
            y = ops.conv2d(x, w1, b1, relu=True, **bound)        # [n, 4*Cout, h, w], channels ordered (a, b, co)
            n, _, h, w = y.shape
            if not (y.is_contiguous(memory_format=torch.channels_last) and y.dim() == 4):
                y = y.reshape(n, 2, 2, cout, h, w).permute(0, 3, 4, 1, 5, 2).reshape(n, cout, 2 * h, 2 * w)
                return ops.conv2d(y, self.mask_score.weight, self.mask_score.bias, out_format="nchw", **bound)
            # The pixel shuffle only permutes pixels and mask_score is a 1x1 conv, so they commute: score the four
            # (a, b) channel groups in place -- the NHWC storage [n,h,w,(a,b,co)] IS an NHWC tensor of 4w "pixels" per
            # row with Cout channels (a free view) -- and shuffle the num_classes-channel logits instead of the
            # 256-channel feature map (two 50 MB permute copies per call in the first version).
            yv = y.permute(0, 2, 3, 1).reshape(n, h, w * 4, cout).permute(0, 3, 1, 2)
        z = ops.conv2d(yv, self.mask_score.weight, self.mask_score.bias, out_format="nhwc", out_dtype=torch.float32,
                       **bound)                                                                   # [n, K, h, 4w]
        K = z.shape[1]
        z = z.permute(0, 2, 3, 1).reshape(n, h, w, 2, 2, K)                                        # (i, j, a, b, k)
        return z.permute(0, 5, 1, 3, 2, 4).reshape(n, K, 2 * h, 2 * w)

    def forward_train(self, feat, rois, prec):
        """Mask logits with device gradients: FPNRoIAlignFunction 14x14 on the fp32 levels, 4 x (3x3 + ReLU), the 2x2
        deconv + ReLU (training.conv_transpose2x2) and the 1x1 score."""
        M = self.roi_pooling.pooled_height
        if rois.shape[0] == 0:
            return feat[0].new_zeros((0, self.mask_score.weight.shape[0], 2 * M, 2 * M))
        x = training.FPNRoIAlignFunction.apply(rois, M, M, self.roi_pooling.spatial_scale, 2, *feat)
        for i in range(1, 5):
            c = getattr(self, "mask_conv%d" % i)
            x = training.conv2d(x, c[0].weight, c[0].bias, padding=1, relu=not self.gn, precision=prec)
            if self.gn:
                x = training.group_norm(x, c[1].weight, c[1].bias, c[1].num_groups, c[1].eps, relu=True)
        d = self.mask_deconv1[0]
        x = training.conv_transpose2x2(x, d.weight, d.bias, relu=True, precision=prec)
        return training.conv2d(x, self.mask_score.weight, self.mask_score.bias, precision=prec)


class FCNSubNet(nn.Module):
    """models/fcn.py:29-73: num_layers x (DeformConvWithOffset + ReLU); channel drop at layer n-2."""

    def __init__(self, in_channels, out_channels, num_layers, with_norm="none"):
        super().__init__()
        assert num_layers >= 2
        self.num_layers = num_layers
        self.gn = with_norm == "group_norm"
        self.conv = nn.ModuleList()
        for i in range(num_layers):
            if i == num_layers - 2:
                layer = DeformConvWithOffset(in_channels, out_channels, 3, stride=1, padding=1, dilation=1)
                in_channels = out_channels
            else:
                layer = DeformConvWithOffset(in_channels, in_channels, 3, stride=1, padding=1, dilation=1)
            norm = [nn.GroupNorm(32, in_channels)] if self.gn else []       # models/fcn.py:49-50
            self.conv.append(nn.Sequential(layer, *norm, nn.ReLU(inplace=True)))
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                m.weight.data.fill_(0)
                m.bias.data.fill_(0)
            elif isinstance(m, DeformConv):
                nn.init.kaiming_normal_(m.weight.data)
                if m.bias is not None:
                    m.bias.data.fill_(0)

    def forward(self, x):
        for i in range(self.num_layers):
            l = self.conv[i][0]
            offset = ops.conv2d(x, l.conv_offset.weight, l.conv_offset.bias, 1, 1, 1, out_format="nchw")
            x = ops.deform_conv(x, offset, l.conv.weight, l.conv.bias, l.conv.stride, l.conv.padding,
                                l.conv.dilation, l.conv.deformable_groups, relu=not self.gn)   # ReLU fused
            if self.gn:
                gn = self.conv[i][1]
                x = ops.group_norm(x, gn.weight, gn.bias, gn.num_groups, gn.eps, relu=True)
        return x

    def forward_train(self, x):
        """forward with device gradients: each DeformConvWithOffset (its autograd Functions), then GN + ReLU through
        training.group_norm or the ReLU alone."""
        for i in range(self.num_layers):
            x = self.conv[i][0](x)
            if self.gn:
                gn = self.conv[i][1]
                x = training.group_norm(x, gn.weight, gn.bias, gn.num_groups, gn.eps, relu=True)
            else:
                x = F.relu(x)
        return x


class FCNHead(nn.Module):
    """models/fcn.py:76-108."""

    def __init__(self, in_channels, num_classes, num_layers, upsample_rate=4, with_norm="none"):
        super().__init__()
        self.fcn_subnet = FCNSubNet(in_channels, 128, num_layers, with_norm)
        self.upsample_rate = upsample_rate
        self.score = nn.Conv2d(512, num_classes, 1)
        nn.init.normal_(self.score.weight.data, 0, 0.01)
        self.score.bias.data.zero_()
        self.overlap_levels = False   # measured: no gain over the serial P2..P5 order (the side-stream fork already fills the gaps)
        self._streams = None
        self._f = None

    def prepare(self):
        w = self.score.weight.detach()
        self._f = [w[:, 128 * l:128 * (l + 1)].contiguous() for l in range(4)]

    def _subnets(self, p2, p3, p4, p5):
        """The four per-level sub-networks.  P4 / P5 have 64 / 16 output tiles -- far fewer than SMs -- so on CUDA they
        run on two extra streams next to the P2 -> P3 chain instead of after it."""
        if not (p2.is_cuda and self.overlap_levels):
            return tuple(self.fcn_subnet(p) for p in (p2, p3, p4, p5))
        cur = torch.cuda.current_stream(p2.device)
        if self._streams is None:
            self._streams = [torch.cuda.Stream(device=p2.device) for _ in range(2)]
        fork = torch.cuda.Event()
        fork.record(cur)
        outs, joins = {}, []
        for st, (name, p) in zip(self._streams, (("p4", p4), ("p5", p5))):
            st.wait_event(fork)
            with torch.cuda.stream(st):
                outs[name] = self.fcn_subnet(p)
                ev = torch.cuda.Event()
                ev.record(st)
            joins.append(ev)
            if not torch.cuda.is_current_stream_capturing():
                outs[name].record_stream(cur)
        o2 = self.fcn_subnet(p2)
        o3 = self.fcn_subnet(p3)
        for ev in joins:
            cur.wait_event(ev)
        return o2, o3, outs["p4"], outs["p5"]

    def forward(self, p2, p3, p4, p5, score_only=False):
        """score_only (static engine): stop at the quarter-resolution score map 'fcn_score' -- the x4 up-sampling is then
        evaluated inside the panoptic fusion kernel (ops.panoptic_fuse(..., up4=True)) and fcn_output is never materialised."""
        p2, p3, p4, p5 = self._subnets(p2, p3, p4, p5)
        if self._f is not None:     # prepared (inference): score each level at its own resolution
            # models/fcn.py:94-101 computes score(cat(p2, up2(p3), up4(p4), up8(p5))).  The 1x1 score conv and the
            # bilinear upsampling are both linear and act on different axes, so they commute:
            #   score = W2*p2 + up2(W3*p3) + up4(W4*p4) + up8(W5*p5) + b
            # -- identical up to fp32 reassociation, and the three 128-channel upsampled maps plus the
            # 512-channel concat (0.5 GB of traffic at 1024x2048) are never built.
            score = ops.conv2d(p2, self._f[0], self.score.bias, out_format="nchw").float()
            parts = [ops.conv2d(feat, self._f[l], None, out_format="nchw").float() for l, feat in enumerate((p3, p4, p5), start=1)]
            if score.is_cuda and score.shape[2] % 8 == 0 and score.shape[3] % 8 == 0 and \
                    all(tuple(s_.shape[2:]) == (score.shape[2] >> l, score.shape[3] >> l) for l, s_ in enumerate(parts, start=1)):
                score = ops.fcn_score_fuse(score, *parts)            # one launch: s2 + up2(s3) + up4(s4) + up8(s5)
            else:
                for l, s_l in enumerate(parts, start=1):
                    score = score + F.interpolate(s_l, None, 2 ** l, mode="bilinear", align_corners=False)
            ret = {"fcn_score": score}
            if self.upsample_rate != 1 and not (score_only and self.upsample_rate == 4):
                ret["fcn_output"] = ops.upsample_bilinear(score, self.upsample_rate)
            return ret
        p3 = F.interpolate(p3, None, 2, mode="bilinear", align_corners=False)
        p4 = F.interpolate(p4, None, 4, mode="bilinear", align_corners=False)
        p5 = F.interpolate(p5, None, 8, mode="bilinear", align_corners=False)
        feat = torch.cat([p2, p3, p4, p5], dim=1)
        score = ops.conv2d(feat, self.score.weight, self.score.bias, out_format="nchw")  # panoptic kernel reads planes
        ret = {"fcn_score": score, "fcn_feat": feat}
        if self.upsample_rate != 1:
            ret["fcn_output"] = F.interpolate(score, None, self.upsample_rate, mode="bilinear", align_corners=False)
        return ret

    def forward_train(self, p2, p3, p4, p5, prec):
        """fcn_score with device gradients, by the prepared forward's commutation: each level through the subnet's
        DeformConvWithOffset layers and its 128-channel slice of the 1x1 score conv, the four maps summed at P2
        resolution by FcnScoreFuseFunction.  The concat and fcn_output are never built (SemanticLoss up-samples)."""
        w = self.score.weight
        scores = []
        for l, feat in enumerate((p2, p3, p4, p5)):
            feat = self.fcn_subnet.forward_train(feat)
            scores.append(training.conv2d(feat, w[:, 128 * l:128 * (l + 1)], self.score.bias if l == 0 else None,
                                          precision=prec))
        return training.FcnScoreFuseFunction.apply(*scores)


# ---------------------------------------------------------------------------------------------
class resnet_upsnet(nn.Module):
    """models/resnet_upsnet.py:38-248 (test branch)."""

    def __init__(self, backbone_depth, cfg=None):
        super().__init__()
        cfg = cfg or UPSNetConfig()
        self.cfg = cfg
        self.num_classes, self.num_seg_classes = cfg.num_classes, cfg.num_seg_classes
        self.num_reg_classes = cfg.num_classes
        _check_norms(cfg)
        _check_fpn_upsample(cfg)
        self.resnet_backbone = ResNetBackbone(backbone_depth, cfg)
        self.fpn = FPN(cfg.fpn_feature_dim, cfg.fpn_with_gap, cfg.fpn_with_norm, cfg.fpn_upsample_method)
        self.rpn = RPN(cfg.num_anchors, cfg.fpn_feature_dim)      # rpn_with_norm unused, as in resnet_upsnet.py:52
        self.rcnn = RCNN(self.num_classes, self.num_reg_classes, dim_in=cfg.fpn_feature_dim, with_norm=cfg.rcnn_with_norm)
        self.mask_branch = MaskBranch(self.num_classes, cfg.mask_size, dim_in=cfg.fpn_feature_dim,
                                      with_norm=cfg.rcnn_with_norm)
        self.fcn_head = FCNHead(cfg.fpn_feature_dim, self.num_seg_classes, cfg.fcn_num_layers,
                                with_norm=cfg.fcn_with_norm)
        self.enable_void = cfg.panoptic_box_keep_fraction < 1
        assert self.enable_void, "all shipped configs enable the void channel"
        self.pyramid_proposal = ProposalGenerator(cfg.rpn_feat_stride, cfg.anchor_scales, cfg.anchor_ratios,
                                                  cfg.rpn_pre_nms_top_n, cfg.rpn_post_nms_top_n,
                                                  cfg.rpn_nms_thresh, cfg.rpn_min_size)
        self.pyramid_proposal_train = ProposalGenerator(cfg.rpn_feat_stride, cfg.anchor_scales, cfg.anchor_ratios,
                                                        cfg.train_rpn_pre_nms_top_n, cfg.train_rpn_post_nms_top_n,
                                                        cfg.train_rpn_nms_thresh, cfg.train_rpn_min_size)
        self.mask_roi = MaskROI(cfg.max_det, self.num_classes, cfg.nms_thresh, False, cfg.score_thresh,
                                cfg.bbox_reg_weights)
        self.mask_roi_panoptic = MaskROI(cfg.max_det, self.num_classes, 0.5, True, cfg.panoptic_score_thresh,
                                         cfg.bbox_reg_weights)
        self.panoptic_head = ops.PanopticHead(self.num_seg_classes, self.num_classes, 0.3)
        # static-shape, sync-free twins used by the engine path (CUDA-graph capturable)
        self.pyramid_proposal_static = StaticProposalGenerator(cfg.rpn_feat_stride, cfg.anchor_scales,
                                                               cfg.anchor_ratios, cfg.rpn_pre_nms_top_n,
                                                               cfg.rpn_post_nms_top_n, cfg.rpn_nms_thresh,
                                                               cfg.rpn_min_size)
        self.mask_roi_static = StaticMaskROI(cfg.max_det, self.num_classes, cfg.nms_thresh, False, cfg.score_thresh,
                                             cfg.bbox_reg_weights)
        self.mask_roi_panoptic_static = StaticMaskROI(cfg.max_det, self.num_classes, 0.5, True,
                                                      cfg.panoptic_score_thresh, cfg.bbox_reg_weights)
        self.static_engine = True     # fixed shapes + device-side counts: no host sync inside the forward
        self.use_cuda_graph = True    # capture the static forward once per (shape, precision) and replay it
        self.overlap_heads = True     # semantic head on a side stream, concurrent with the detection chain
        self.dedup_mask_rows = True   # mask branch on the distinct boxes only (ops.mask_rows), not on both padded buffers
        self._side = {}
        self._graphs = {}
        self._pools = {}
        # captured graphs kept (LRU), one per (padded input shape, precision, lane).  The graphs of a lane share one
        # activation pool, so an entry costs its graph and static outputs plus what its shape adds to the pool: a median
        # of 53 MB (bf16x3) / 64 MB (bf16), at most 432 MB, of memory_reserved for COCO R50 shapes up to 800x1344 on an
        # H100 80GB HBM3 at 700 W (scripts/prof_mixed_sizes.py).  128 keeps a COCO-style mix (35 padded shapes in 120 images) resident on 2 lanes.
        self.max_graphs = 128
        self._prepared = False
        self.eval()
        # backbone_freeze_at and backbone_fix_bn (models/resnet.py:69-78, 338-345): the stem, res2..res<freeze_at> and,
        # with fix_bn, every BatchNorm are frozen, so they get no gradient and get_params_lr() does not list them
        bb = self.resnet_backbone
        frozen = [bb.conv1] + [getattr(bb, "res%d" % i) for i in range(2, cfg.backbone_freeze_at + 1)]
        if cfg.backbone_fix_bn:
            frozen += [m for m in self.modules() if isinstance(m, nn.BatchNorm2d)]
        for m in frozen:
            for p in m.parameters():
                p.requires_grad_(False)

    def prepare(self):
        """Fold frozen BN, fuse sibling 1x1 heads, reshape the deconv: call after loading weights."""
        ops.forget_packed(self.parameters())
        for m in self.modules():
            if m is not self and hasattr(m, "prepare"):
                m.prepare()
        self._prepared = True
        return self

    def _apply(self, fn, *a, **kw):
        """.to() / .cuda() / .float(): the folded / fused weights made by prepare() and the captured graphs refer to the
        old parameter storage -- rebuild them lazily on the next forward."""
        r = super()._apply(fn, *a, **kw)
        self._prepared = False
        self._graphs, self._pools = {}, {}
        return r

    # COCO -> Cityscapes head remapping of models/resnet.py:223-273 (fine-tuning a COCO checkpoint on Cityscapes)
    _COCO2CITY_THING = {0: 0, 1: 1, 2: -1, 3: 3, 4: 8, 5: 6, 6: 7, 7: 4, 8: 2}
    _COCO2CITY_SEG = {0: 20, 1: 43, 2: 49, 3: 51, 4: 37, 5: -1, 6: 62, 7: -1, 8: 36, 9: -1, 10: 39, 11: 53, 12: -1, 13: 55,
                      14: 60, 15: 58, 16: 59, 17: 56, 18: 54}

    @staticmethod
    def name_mapping(name, resume=False):
        """models/resnet.py:213-222: checkpoints of this model (`resume`) may carry DataParallel's `module.` prefix;
        backbone-only checkpoints use torchvision / caffe names (conv1, bn1, layer1..4)."""
        if resume:
            return name[len("module."):] if name.startswith("module.") else name
        if name.startswith("conv1") or name.startswith("bn1"):
            return "resnet_backbone.conv1." + name
        return name.replace("layer1", "resnet_backbone.res2.layers").replace("layer2", "resnet_backbone.res3.layers") \
                   .replace("layer3", "resnet_backbone.res4.layers").replace("layer4", "resnet_backbone.res5.layers")

    def load_state_dict(self, state_dict, strict=True, resume=None, **kw):
        """nn.Module.load_state_dict, or -- when `resume` is given, the way upsnet_end2end_test.py:190-193 and the
        training scripts call it -- the reference's own loader (models/resnet.py:224-299): key remapping, the COCO ->
        Cityscapes head conversion, shape-checked copies with warnings instead of errors."""
        if resume is None:
            r = super().load_state_dict(state_dict, strict=strict, **kw)
        else:
            r = self._load_reference_style(dict(state_dict), bool(resume))
        self._prepared = False
        self._graphs, self._pools = {}, {}
        return r

    def _load_reference_style(self, state_dict, resume):
        import warnings
        own = self.state_dict()
        k = "rcnn.cls_score.weight"
        if k in state_dict and own[k].shape[0] == 9 and state_dict[k].shape[0] == 81:          # resnet.py:227-250
            for wn in ("rcnn.cls_score.weight", "rcnn.cls_score.bias", "rcnn.bbox_pred.weight", "rcnn.bbox_pred.bias",
                       "mask_branch.mask_score.weight", "mask_branch.mask_score.bias"):
                src = state_dict[wn].float()
                mean, std = src.mean().item(), src.std().item()
                src = src.view(*([81, -1] + list(src.shape[1:])))
                blobs = (np.random.randn(*([9] + list(src.shape[1:]))) * std + mean).astype(np.float32)
                for i in range(9):
                    c = self._COCO2CITY_THING[i]
                    if c >= 0:
                        blobs[i] = src[c].cpu().numpy()
                state_dict[wn] = torch.from_numpy(blobs.reshape([-1] + list(src.shape[2:])))
        k = "fcn_head.score.weight"
        if k in own and k in state_dict and own[k].shape[0] == 19 and state_dict[k].shape[0] == 133:   # resnet.py:252-283
            for wn in ("fcn_head.score.weight", "fcn_head.score.bias"):
                src = state_dict[wn].float()
                mean, std = src.mean().item(), src.std().item()
                blobs = (np.random.randn(*([19] + list(src.shape[1:]))) * std + mean).astype(np.float32)
                for i in range(19):
                    c = self._COCO2CITY_SEG[i]
                    if c >= 0:
                        blobs[i] = src[c].cpu().numpy()
                state_dict[wn] = torch.from_numpy(blobs)
        seen = set()
        with torch.no_grad():
            for name, param in state_dict.items():
                name = self.name_mapping(name, resume)
                seen.add(name)
                if name not in own:
                    warnings.warn('unexpected key "{}" in state_dict'.format(name))
                    continue
                if own[name].shape == param.shape:
                    own[name].copy_(param)
                else:
                    warnings.warn("While copying the parameter named {}, whose dimensions in the models are {} and whose "
                                  "dimensions in the checkpoint are {}, ...".format(name, own[name].size(), param.size()))
        missing = set(own.keys()) - seen
        if missing:
            warnings.warn('missing keys in state_dict: "{}"'.format(missing))
        return None

    # ------------------------------------------------------------------------------------------
    # static engine: every tensor has a fixed shape, counts stay on the device
    # ------------------------------------------------------------------------------------------
    def _forward_static(self, x, im_info):
        res2, res3, res4, res5 = self.resnet_backbone(x)
        p2, p3, p4, p5, p6 = self.fpn(res2, res3, res4, res5)
        rpn_cls_prob, rpn_bbox_pred = [], []
        for feat in (p2, p3, p4, p5, p6):
            _, bbox, prob = self.rpn(feat)
            rpn_cls_prob.append(prob)
            rpn_bbox_pred.append(bbox)
        # The semantic head (8 offset convs + 8 deformable convs, machine-filling kernels) does not depend on the
        # detection chain (top-k, NMS sweeps, MaskROI: single-CTA, latency-bound kernels): fork it onto a side stream
        # and join before the panoptic head, so the small kernels hide under the big ones (also inside the CUDA graph).
        fork = x.is_cuda and self.overlap_heads
        if fork:
            cur = torch.cuda.current_stream(x.device)
            side = self._side_stream(x.device)
            ev = torch.cuda.Event()
            ev.record(cur)
            side.wait_event(ev)
            with torch.cuda.stream(side):
                fcn_output, fcn_score = self._semantic(p2, p3, p4, p5, x.is_cuda)
                done = torch.cuda.Event()
                done.record(side)
            if not torch.cuda.is_current_stream_capturing():
                for t_ in (fcn_output, fcn_score):      # eager mode: consumed on `cur` (graph pools need no hint)
                    if t_ is not None:
                        t_.record_stream(cur)
        rois, _, roi_valid = self.pyramid_proposal_static(rpn_cls_prob, rpn_bbox_pred, im_info)
        if not fork:
            fcn_output, fcn_score = self._semantic(p2, p3, p4, p5, x.is_cuda)
        feats = [p2, p3, p4, p5]
        rcnn_output = self.rcnn(feats, rois)
        cls_prob = F.softmax(rcnn_output["cls_score"].float(), dim=1)
        bbox_pred = rcnn_output["bbox_pred"].float()
        # the two MaskROIs (detections / panoptic candidates) are independent chains of single-CTA kernels: run the second
        # on its own stream next to the first
        if fork:
            side2 = self._side_stream(x.device, 1)
            ev2 = torch.cuda.Event()
            ev2.record(cur)
            side2.wait_event(ev2)
            with torch.cuda.stream(side2):
                s2, b2, c2, n2 = self.mask_roi_panoptic_static(rois, roi_valid, bbox_pred, cls_prob, im_info, side=True)
                done2 = torch.cuda.Event()
                done2.record(side2)
            if not torch.cuda.is_current_stream_capturing():
                for t_ in (s2, b2, c2, n2, self.mask_roi_panoptic_static.last_flags):
                    t_.record_stream(cur)
        s1, b1, c1, n1 = self.mask_roi_static(rois, roi_valid, bbox_pred, cls_prob, im_info)
        if fork:
            cur.wait_event(done2)
        else:
            s2, b2, c2, n2 = self.mask_roi_panoptic_static(rois, roi_valid, bbox_pred, cls_prob, im_info)
        # models/resnet_upsnet.py:203-222 runs the mask branch twice (detections, panoptic candidates).  Every roi is
        # processed independently, so both sets go through it as ONE batch: half the launches, fuller tile waves.
        # A roi's logits depend on its box alone, and a candidate that also survives as a detection has the detection's
        # box bit for bit (same maskroi_prepare decode), so the batch is the u distinct live boxes: the detections, then
        # the candidates that match none (ops.mask_rows).  The branch skips rows >= u, so mask_probs rows >= n1 are
        # unspecified.
        ms = self.cfg.mask_size
        if self.dedup_mask_rows and x.is_cuda:
            rows, u, pan_row = ops.mask_rows(b1, n1, b2, n2)
            logits = self.mask_branch(feats, rows, n_dev=u).float()
            K = logits.shape[1]
            mask_score = logits.view(-1, ms, ms).index_select(0, pan_row.long() * K + c2).view(-1, 1, ms, ms)
        else:
            logits = self.mask_branch(feats, torch.cat([b1, b2], 0)).float()
            mask_score = logits[b1.shape[0]:].gather(1, c2.view(-1, 1, 1, 1).expand(-1, -1, ms, ms))
        mask_prob = torch.sigmoid(logits[:b1.shape[0]])
        if fork:
            cur.wait_event(done)
        # fused x4 up-sampling: the fusion kernel reads the quarter-resolution score map (fcn_output, when the parity tests ask
        # for it, is the same arithmetic materialised by the stand-alone kernel)
        keep, labels, sem, k = ops.panoptic_fuse(fcn_score if fcn_score is not None else fcn_output, b2[:, 1:], s2, mask_score, c2,
                                                 self.panoptic_head.num_stuff, self.panoptic_head.fraction_threshold,
                                                 want_sem=True, n_dev=n2.reshape(1), up4=fcn_score is not None)
        counts = torch.cat([n1.reshape(1).to(torch.int32), n2.reshape(1).to(torch.int32), k.reshape(1)])
        # != 0 when a static MaskROI buffer dropped detections the reference would have kept (see StaticMaskROI.last_flags)
        trunc = torch.stack([self.mask_roi_static.last_flags.reshape(()).to(torch.int32),
                             self.mask_roi_panoptic_static.last_flags.reshape(()).to(torch.int32)])
        out = {"cls_probs": s1, "pred_boxes": b1, "mask_probs": mask_prob, "cls_inds": c1, "fcn_outputs": sem,
               "panoptic_outputs": labels, "p_scores": s2, "p_cls": c2, "p_boxes": b2, "p_mask_score": mask_score,
               "keep": keep, "counts": counts, "trunc_flags": trunc, "fcn_output": fcn_output}
        if getattr(self, "keep_intermediates", False):   # parity tests against the literal oracle: every stage boundary
            out["dbg"] = {"fpn": [f.float().contiguous() for f in (p2, p3, p4, p5, p6)],
                          "rpn_cls_prob": [t_.float() for t_ in rpn_cls_prob], "rpn_bbox_pred": [t_.float() for t_ in rpn_bbox_pred],
                          "rois": rois, "roi_valid": roi_valid, "cls_score": rcnn_output["cls_score"].float(),
                          "bbox_pred": bbox_pred, "mask_logits": logits}
        return out

    def _semantic(self, p2, p3, p4, p5, on_gpu=True):
        """Semantic head of the static engine: (fcn_output or None, fcn_score or None).  With the fused score path and the
        reference's x4 up-sampling the full-resolution logits are only materialised when a test asks for intermediates."""
        head = self.fcn_head
        fuse_up = on_gpu and head._f is not None and head.upsample_rate == 4
        if not fuse_up:
            return head(p2, p3, p4, p5)["fcn_output"].float(), None
        ret = head(p2, p3, p4, p5, score_only=not getattr(self, "keep_intermediates", False))
        score = ret["fcn_score"].float().contiguous()
        fo = ret.get("fcn_output")
        return (None if fo is None else fo.float()), score

    def _side_stream(self, dev, idx=0):
        key = (str(dev), idx, ops.WS_SLOT["i"])
        if key not in self._side:
            self._side[key] = torch.cuda.Stream(device=dev)
        return self._side[key]

    def _run_static(self, x, im_info, lane=0):
        """One image through the static engine on the CURRENT stream.  im_info: the image's (h, w, scale) row, a host row
        or a CUDA float32 [3] tensor.  `lane` selects an independent engine instance (its own captured graphs, activation
        pool, output buffers and scratch workspaces): callers that keep several images in flight run lane i on stream i
        (pipeline.PipelinedEngine, bench.py) -- the single-CTA detection kernels of one image then hide under the
        machine-filling convolutions of the other."""
        prev_slot = ops.WS_SLOT["i"]
        ops.WS_SLOT["i"] = int(lane)
        try:
            return self._run_static_lane(x, im_info, int(lane))
        finally:
            ops.WS_SLOT["i"] = prev_slot

    @staticmethod
    def _write_im_info(ent, im_info):
        """Enqueue the copy of im_info into the entry's device row on the current stream.  A host row is staged in pinned
        memory (torch's pinned allocator holds the block until the copy has run), so the host never waits; it is not
        copied again while it equals the row last written to this entry."""
        if torch.is_tensor(im_info) and im_info.is_cuda:
            ent[4].copy_(im_info.reshape(3), non_blocking=True)
            ent[5] = None
            return
        row = tuple(np.asarray(im_info, dtype=np.float32).reshape(-1)[:3].tolist())
        if row != ent[5]:
            ent[4].copy_(torch.tensor(row, dtype=torch.float32).pin_memory(), non_blocking=True)
            ent[5] = row

    def _run_static_lane(self, x, im_info, lane):
        if not (self.use_cuda_graph and x.is_cuda):
            return self._forward_static(x, ops.im_info_device(im_info, x.device)), None
        # the image geometry is a device input of the graph (the detection clips read it when they run), so one graph
        # serves every image of a padded shape
        key = (tuple(x.shape), str(x.device), ops._PRECISION["conv"], bool(getattr(self, "keep_intermediates", False)),
               bool(self.dedup_mask_rows), lane)
        ent = self._graphs.get(key)
        if ent is None:
            static_x = torch.empty(x.shape, dtype=torch.float32, device=x.device)
            static_x.copy_(x)
            ent = [None, static_x, None, 0, torch.empty((3,), dtype=torch.float32, device=x.device), None]
            self._write_im_info(ent, im_info)
            cur = torch.cuda.current_stream(x.device)
            side = torch.cuda.Stream(device=x.device)
            side.wait_stream(cur)
            with torch.cuda.stream(side):       # warm-up: workspaces, packed weights, anchor tables, cudnn/cub plans
                for _ in range(2):
                    self._forward_static(static_x, ent[4])
            cur.wait_stream(side)
            torch.cuda.synchronize(x.device)
            # Every graph of a lane is captured into the lane's one memory pool, so k captured shapes cost about one
            # activation pool.  Their intermediates overlap, which is safe under one invariant: a lane's graphs never
            # replay concurrently (a lane runs on one stream), and a graph's outputs are consumed -- copied or cloned,
            # as _forward_infer and PipelinedEngine do -- before the lane replays any graph again.
            pool = self._pools.get((str(x.device), lane))
            if pool is None:
                pool = self._pools[(str(x.device), lane)] = torch.cuda.graph_pool_handle()
            graph = torch.cuda.CUDAGraph()
            l0 = ops.STATS["launches"]
            with torch.cuda.graph(graph, pool=pool):
                out = self._forward_static(static_x, ent[4])
            ent[0], ent[2], ent[3] = graph, out, ops.STATS["launches"] - l0
            while len(self._graphs) >= self.max_graphs:      # LRU
                self._graphs.pop(next(iter(self._graphs)))
            self._graphs[key] = ent
        else:
            self._graphs[key] = self._graphs.pop(key)        # most recently used last
            ent[1].copy_(x, non_blocking=True)
            self._write_im_info(ent, im_info)
        graph, _, out, n_launch = ent[:4]
        graph.replay()
        ops.STATS["launches"] += n_launch
        return out, graph

    def get_params_lr(self):
        """The reference's 13 parameter groups (models/resnet_upsnet.py:260-285, get_params of models/resnet.py:31-51):
        the GroupNorm group (every nn.GroupNorm's weight and bias, at lr 1 without weight decay; empty without
        group_norm), then for res3-res5, fpn, rcnn, mask_branch, rpn and fcn_head the weights at lr 1 and the biases at
        lr 2 without weight decay, selected by the same name rule, with the GroupNorm parameters excluded except from
        the rpn groups (the reference does not exclude them there; its RPN never has any).  Only parameters with
        requires_grad, except in the GroupNorm group, which the reference does not filter."""
        gn_params, gn_names = [], set()
        for n, m in self.named_modules():
            if isinstance(m, nn.GroupNorm):
                gn_params += [m.weight, m.bias]
                gn_names |= {n + ".weight", n + ".bias"}

        def params(prefixes, suffix, exclude=()):
            for name, module in self.named_modules():
                if name in prefixes:
                    for n, p in module.named_parameters():
                        n = name + "." + n
                        if n in exclude:
                            continue
                        if (n.split(".")[-1].startswith(suffix) or n.endswith(suffix)) and p.requires_grad:
                            yield p
        groups = [{"params": gn_params, "lr": 1, "weight_decay": 0}]
        for prefixes in (["resnet_backbone.res3", "resnet_backbone.res4", "resnet_backbone.res5"], ["fpn"], ["rcnn"],
                         ["mask_branch"], ["rpn"], ["fcn_head"]):
            ex = gn_names if prefixes[0] in ("fpn", "rcnn", "mask_branch", "fcn_head") else ()
            groups.append({"params": list(params(prefixes, "weight", ex)), "lr": 1})
            groups.append({"params": list(params(prefixes, "bias", ex)), "lr": 2, "weight_decay": 0})
        return groups

    def forward(self, data, label=None):
        """Inference (label None): the reference's result dict.  Training (label = the reference loader's dict): the
        nine losses and accuracies of models/resnet_upsnet.py:180-193, each float32 [1] on the device, differentiable in
        every parameter get_params_lr() lists (see _forward_train)."""
        if label is not None:
            return self._forward_train(data, label)
        with torch.no_grad():
            return self._forward_infer(data)

    def _forward_infer(self, data):
        if not self._prepared:
            self.prepare()
        x = data["data"]
        im_info = np.asarray(data["im_info"], dtype=np.float32).reshape(-1, 3)
        assert x.shape[0] == 1 and im_info.shape[0] == 1, "one image per device (SURVEY F9)"
        if self.static_engine:
            out, graph = self._run_static(x, im_info[0])
            n1, n2, k = (int(v) for v in out["counts"].tolist())       # the one host read: result sizes
            keep = out["keep"][:k]
            cp = (lambda t: t.clone()) if graph is not None else (lambda t: t)   # graph buffers are reused
            results = {"cls_probs": cp(out["cls_probs"][:n1]), "pred_boxes": cp(out["pred_boxes"][:n1]),
                       "mask_probs": cp(out["mask_probs"][:n1]), "cls_inds": cp(out["cls_inds"][:n1]),
                       "fcn_outputs": cp(out["fcn_outputs"]), "panoptic_cls_inds": out["p_cls"][:n2][keep],
                       "panoptic_cls_probs": out["p_scores"][:n2][keep], "panoptic_outputs": cp(out["panoptic_outputs"])}
            if getattr(self, "keep_intermediates", False):
                results["_intermediates"] = {"fcn_output": cp(out["fcn_output"]), "pmask_rois": cp(out["p_boxes"][:n2]),
                                             "pcls_prob": cp(out["p_scores"][:n2]),
                                             "pmask_score": cp(out["p_mask_score"][:n2]),
                                             "pcls_idx": cp(out["p_cls"][:n2]), "keep_inds": cp(keep)}
                for k_, v_ in out.get("dbg", {}).items():
                    results["_intermediates"][k_] = [cp(t_) for t_ in v_] if isinstance(v_, list) else cp(v_)
            return results
        res2, res3, res4, res5 = self.resnet_backbone(x)
        p2, p3, p4, p5, p6 = self.fpn(res2, res3, res4, res5)
        rpn_cls_prob, rpn_bbox_pred = [], []
        for feat in (p2, p3, p4, p5, p6):
            _, bbox, prob = self.rpn(feat)
            rpn_cls_prob.append(prob)
            rpn_bbox_pred.append(bbox)
        rois, _ = self.pyramid_proposal(rpn_cls_prob, rpn_bbox_pred, im_info[0])
        fcn_output = self.fcn_head(p2, p3, p4, p5)
        feats = [p2, p3, p4, p5]
        rcnn_output = self.rcnn(feats, rois)
        cls_prob = F.softmax(rcnn_output["cls_score"], dim=1)
        bbox_pred = rcnn_output["bbox_pred"]

        cls_prob_all, mask_rois, cls_idx = self.mask_roi(rois, bbox_pred, cls_prob, im_info[0])
        mask_prob = torch.sigmoid(self.mask_branch(feats, mask_rois))
        results = {"cls_probs": cls_prob_all, "pred_boxes": mask_rois, "mask_probs": mask_prob, "cls_inds": cls_idx}

        # ---- panoptic head (resnet_upsnet.py:217-247) ----
        pcls_prob, pmask_rois, pcls_idx = self.mask_roi_panoptic(rois, bbox_pred, cls_prob, im_info[0])
        mask_score = self.mask_branch(feats, pmask_rois)
        ms = self.cfg.mask_size
        mask_score = mask_score.gather(1, pcls_idx.view(-1, 1, 1, 1).expand(-1, -1, ms, ms))
        pan = self.panoptic_head(fcn_output["fcn_output"], pmask_rois, pcls_prob, mask_score, pcls_idx, want_sem=True)
        keep = pan["keep_inds"]
        results.update({"fcn_outputs": pan["fcn_outputs"], "panoptic_cls_inds": pcls_idx[keep],
                        "panoptic_cls_probs": pcls_prob[keep], "panoptic_outputs": pan["panoptic_outputs"]})
        if getattr(self, "keep_intermediates", False):   # parity tests: the exact inputs of the panoptic head
            results["_intermediates"] = {"fcn_output": fcn_output["fcn_output"], "rois": rois, "cls_prob": cls_prob,
                                         "bbox_pred": bbox_pred, "pmask_rois": pmask_rois, "pcls_prob": pcls_prob,
                                         "pmask_score": mask_score, "pcls_idx": pcls_idx, "keep_inds": keep}
        return results

    # ------------------------------------------------------------------------------------------
    # training forward: eager autograd, separate from the static engine
    # ------------------------------------------------------------------------------------------
    def _forward_train(self, data, label):
        """models/resnet_upsnet.py:88-195 with label (one image).

        Each module runs its forward_train: the backbone with conv1 and res2 frozen on the inference path
        (backbone_freeze_at = 2), then the FPN (with its global-context branch under fpn_with_gap), the RPN per level, the semantic head, the RCNN and the mask branch, with device gradients.  Proposals, proposal targets and the
        panoptic keep draw run without gradients; np.random governs their draws, as in the reference, so the modules
        run in the order below.  With train.fcn_with_roi_loss, the semantic head's ROI loss (FcnRoiLoss) runs on every
        ground-truth box, taken before the keep draw as the reference takes them; the label must then carry
        seg_roi_gt with one row per such box, which is checked before anything is launched.  With keep_intermediates the
        output also carries those boxes ('fcn_rois').

        Precision follows set_precision: 'bf16' runs the training convs in bf16; 'bf16x3' and 'fp32' run them in bf16x3
        (there is no fp32 tensor-core backward).  A training forward drops the folded weights and captured graphs of the
        inference engine, so the next inference forward folds the updated parameters again."""
        cfg = self.cfg
        if cfg.fcn_with_roi_loss:
            self._check_seg_roi_gt(label)
        if cfg.backbone_freeze_at != 2 or not cfg.backbone_fix_bn:
            raise _lib.UpsnetError("training forward: only backbone_freeze_at = 2 with backbone_fix_bn (every shipped "
                                   "configuration) is built, not freeze_at = %d, fix_bn = %s"
                                   % (cfg.backbone_freeze_at, cfg.backbone_fix_bn))
        x = data["data"]
        _lib.require_cuda(x)
        im_info = np.asarray(data["im_info"].cpu() if torch.is_tensor(data["im_info"]) else data["im_info"],
                             dtype=np.float32).reshape(-1, 3)
        if x.shape[0] != 1 or im_info.shape[0] != 1:
            raise _lib.UpsnetError("training forward: one image per device")
        # the optimiser updates the parameters in place after this step, possibly from a replayed CUDA graph
        self._prepared = False
        self._graphs = {}
        ops.forget_packed(self.parameters())
        dev = x.device
        prec = "bf16" if ops._PRECISION["conv"] == _lib.PREC_BF16 else "bf16x3"
        lab = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in label.items()}

        r2, r3, r4, r5 = self.resnet_backbone.forward_train(x, prec)
        p2, p3, p4, p5, p6 = self.fpn.forward_train(r2, r3, r4, r5, prec)
        rpn_score, rpn_bbox = [], []
        for feat in (p2, p3, p4, p5, p6):
            score, bbox = self.rpn.forward_train(feat, prec)
            rpn_score.append(score)
            rpn_bbox.append(bbox)
        with torch.no_grad():
            rois, _ = self.pyramid_proposal_train([torch.sigmoid(s.detach()) for s in rpn_score], [b.detach() for b in rpn_bbox], im_info[0])
            targets = training.ProposalTargets(num_classes=self.num_reg_classes, batch_rois=cfg.batch_rois,
                                               fg_fraction=cfg.fg_fraction, bbox_reg_weights=cfg.bbox_reg_weights,
                                               mask_size=cfg.mask_size).from_roidb(rois, lab["roidb"], im_info)
        (s_rois, cls_label, bbox_target, bbox_iw, bbox_ow, mask_rois, mask_target, _, _) = targets
        fcn_score = self.fcn_head.forward_train(p2, p3, p4, p5, prec)

        # instance head
        levels = [p2, p3, p4, p5]
        cls_score, bbox_pred = self.rcnn.forward_train(levels, s_rois, prec)
        mask_score = self.mask_branch.forward_train(levels, mask_rois, prec)
        cls_loss, bbox_loss, mask_loss, rcnn_acc = training.MaskRCNNLoss(cfg.batch_rois)(
            cls_score, bbox_pred, mask_score, cls_label, bbox_target, bbox_iw, bbox_ow, mask_target)
        rpn_cls_loss, rpn_bbox_loss = training.RPNLoss(rpn_batch_size=cfg.rpn_batch_size)(rpn_score, rpn_bbox, lab)
        fcn_loss = training.SemanticLoss()(fcn_score, lab["seg_gt"])

        # panoptic head on the ground-truth boxes; the ROI loss takes all of them, before the keep draw
        gt_rois, cls_idx = training.gt_rois(lab["roidb"], im_info[0, 2], dev)
        fcn_rois = gt_rois
        if cfg.fcn_with_roi_loss:
            fcn_roi_loss = training.FcnRoiLoss(cfg.mask_size)(fcn_score, self.fcn_head.score.bias, fcn_rois,
                                                              lab["seg_roi_gt"])
        keep = training.draw_keep(gt_rois.shape[0], cfg.panoptic_box_keep_fraction) if self.enable_void else None
        if keep is not None:
            kd = torch.from_numpy(keep).to(dev)
            gt_rois, cls_idx = gt_rois[kd], cls_idx[kd]
        pan_mask = self.mask_branch.forward_train(levels, gt_rois, prec)
        pan = training.PanopticLoss(num_seg_classes=self.num_seg_classes, num_classes=self.num_classes,
                                    enable_void=self.enable_void, mask_size=cfg.mask_size)
        panoptic_loss, panoptic_acc = pan(fcn_score, pan_mask, gt_rois, cls_idx, lab["seg_gt_4x"], lab["mask_gt"], keep)

        out = {"rpn_cls_loss": rpn_cls_loss, "rpn_bbox_loss": rpn_bbox_loss, "cls_loss": cls_loss, "bbox_loss": bbox_loss,
               "mask_loss": mask_loss, "fcn_loss": fcn_loss, "panoptic_loss": panoptic_loss, "rcnn_accuracy": rcnn_acc,
               "panoptic_accuracy": panoptic_acc}
        out = {k: v.reshape(1) for k, v in out.items()}
        if cfg.fcn_with_roi_loss:
            out["fcn_roi_loss"] = fcn_roi_loss
        if getattr(self, "keep_intermediates", False):   # the discrete decisions of the step, for an oracle replay
            out["_intermediates"] = {
                "rois": rois, "proposal_targets": dict(zip(training.ProposalTargets.NAMES, targets)), "gt_rois": gt_rois,
                "cls_idx": cls_idx, "keep_inds": keep, "fpn": [f.detach() for f in (p2, p3, p4, p5, p6)]}
            if cfg.fcn_with_roi_loss:
                out["_intermediates"]["fcn_rois"] = fcn_rois
        return out

    @staticmethod
    def _check_seg_roi_gt(label):
        """fcn_with_roi_loss needs label['seg_roi_gt'] with one [M,M] row per ground-truth box of get_gt_rois
        (non-crowd, class > 0)."""
        roidb = label.get("roidb", {})
        seg = label.get("seg_roi_gt")
        if seg is None or "gt_classes" not in roidb or "is_crowd" not in roidb:
            raise _lib.UpsnetError("training forward: train.fcn_with_roi_loss needs label['seg_roi_gt'] and the roidb's "
                                   "gt_classes / is_crowd")
        n = int(((np.asarray(roidb["gt_classes"]) > 0) & (np.asarray(roidb["is_crowd"]) == 0)).sum())
        if seg.dim() != 3 or seg.shape[0] != n:
            raise _lib.UpsnetError("training forward: train.fcn_with_roi_loss: label['seg_roi_gt'] has %s rows, the "
                                   "roidb %d ground-truth boxes" % (tuple(seg.shape), n))


def resnet_50_upsnet(cfg=None):
    return resnet_upsnet([3, 4, 6, 3], cfg)


def resnet_101_upsnet(cfg=None):
    return resnet_upsnet([3, 4, 23, 3], cfg)
