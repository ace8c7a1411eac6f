"""Training-side pieces of the hot path (BASELINE config #4: UPSNet-50 end2end_train, bf16, 8 GPUs, NCCL all-reduce):

* autograd Functions for the custom operators with hand-written sm_90a BACKWARD kernels (csrc/backward.cu):
    DeformConvFunction / ModDeformConvFunction   operators/functions/deform_conv.py:26-108, mod_deform_conv.py:25-118
    RoIAlignFunction                             operators/functions/roialign.py:21-58
    FPNRoIAlignFunction                          operators/modules/fpn_roi_align.py:32-62 (four RoIAlignFunction calls)
  The dense GEMMs of the deformable backward (d(weight) = dY col^T, d(col) = W^T dY) are library calls (torch.mm), like the
  reference's; the gather / scatter / coordinate-gradient kernels are ours.  OffsetConvFunction makes the offset conv of
  the *WithOffset* modules differentiable; its backward convs are library calls too.
* FlatBucketAllReduce: the gradient all-reduce of `upsnet_end2end_train.py:121` (hvd.DistributedOptimizer) as flat bf16
  buckets over torch.distributed (NCCL between the GPUs, gloo in the CPU tests): gradients are packed per bucket,
  reduced asynchronously while the rest of backward runs, averaged and unpacked before the optimiser step.
* RPNTargets: the RPN training targets of one image (rpn/assign_anchor.py:370-595 add_rpn_blobs / _get_rpn_blobs, run by
  the reference's data loaders on the host) on the device (csrc/rpn_target.cu), as the label dict coco.py:133-142 builds.
* ProposalTargets: the Mask R-CNN proposal targets of one image (operators/modules/proposal_mask_target.py, run by the
  reference on the host in the middle of the forward) on the device (csrc/proposal_target.cu): roi sampling, box
  targets and the class-specific polygon mask targets.

Scope note: this is the operator / communication layer of the training configuration plus the RPN and proposal targets.
Losses and the optimiser are plain torch in the reference and stay that way; the dense backward convolutions are
library calls.
"""
import ctypes as C

import numpy as np
import torch
import torch.distributed as dist
from torch.nn.modules.utils import _pair

from . import _lib
from ._lib import check, f32c, lib, ptr, require_cuda, stream_ptr


def _conv_out(n, pad, dil, k, stride):
    return (n + 2 * pad - (dil * (k - 1) + 1)) // stride + 1


class _DeformConvBase(torch.autograd.Function):
    @staticmethod
    def _geom(x, weight, stride, padding, dilation):
        sh, sw = _pair(stride); ph, pw = _pair(padding); dh, dw = _pair(dilation)
        N, Cin, H, W = x.shape
        Cout, _, kh, kw = weight.shape
        return (N, Cin, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, _conv_out(H, ph, dh, kh, sh), _conv_out(W, pw, dw, kw, sw))

    @staticmethod
    def _forward(ctx, x, offset, mask, weight, bias, stride, padding, dilation):
        from . import operators as ops
        require_cuda(x, offset, weight, bias, mask)
        ctx.save_for_backward(x, offset, mask if mask is not None else x.new_empty(0), weight)
        ctx.has_mask, ctx.has_bias = mask is not None, bias is not None
        ctx.conv = (stride, padding, dilation)
        # fp32 CUDA-core tiles: the training forward keeps fp32 semantics of the reference (.data<float>())
        return ops.deform_conv(x, offset, weight, bias, stride, padding, dilation, 1, mask=mask, precision=_lib.PREC_FP32_SIMT)

    @staticmethod
    def _backward(ctx, grad_out):
        x, offset, mask, weight = ctx.saved_tensors
        mask = mask if ctx.has_mask else None
        stride, padding, dilation = ctx.conv
        N, Cin, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, Ho, Wo = _DeformConvBase._geom(x, weight, stride, padding, dilation)
        x, offset, grad_out = f32c(x), f32c(offset), f32c(grad_out)
        mask = None if mask is None else f32c(mask)
        dev = x.device
        K, P = Cin * kh * kw, Ho * Wo
        w2 = weight.reshape(Cout, K).float()
        dx = torch.empty_like(x)
        doff = torch.empty_like(offset)
        dmask = torch.empty_like(mask) if mask is not None else None
        dw_ = torch.zeros((Cout, K), dtype=torch.float32, device=dev)
        col = torch.empty((K, P), dtype=torch.float32, device=dev)
        g = (Cin, H, W, kh, kw, sh, sw, ph, pw, dh, dw)
        st = stream_ptr(dev)
        with torch.cuda.device(dev):
            for n in range(N):          # the reference loops over the batch as well (functions/deform_conv.py:84-104)
                m_n = None if mask is None else mask[n]
                go = grad_out[n].reshape(Cout, P)
                check(lib().upsnet_dcn_im2col(ptr(x[n]), ptr(offset[n]), ptr(m_n), *g, ptr(col), st), "dcn_im2col")
                dw_.addmm_(go, col.t())                                         # d(weight) += dY col^T
                dcol = torch.mm(w2.t(), go)                                     # d(col) = W^T dY
                check(lib().upsnet_dcn_col2im(ptr(dcol), ptr(offset[n]), ptr(m_n), *g, ptr(dx[n]), st), "dcn_col2im")
                check(lib().upsnet_dcn_col2im_coord(ptr(dcol), ptr(x[n]), ptr(offset[n]), ptr(m_n), *g, ptr(doff[n]),
                                                    ptr(None if dmask is None else dmask[n]), st), "dcn_col2im_coord")
        dbias = grad_out.sum(dim=(0, 2, 3)) if ctx.has_bias else None
        return dx, doff, dmask, dw_.view_as(weight), dbias


class DeformConvFunction(_DeformConvBase):
    """y = DeformConv(x, offset; weight, bias) with hand-written backward kernels (K1-K3)."""

    @staticmethod
    def forward(ctx, x, offset, weight, bias=None, stride=1, padding=0, dilation=1):
        return _DeformConvBase._forward(ctx, x, offset, None, weight, bias, stride, padding, dilation)

    @staticmethod
    def backward(ctx, grad_out):
        dx, doff, _, dw_, db = _DeformConvBase._backward(ctx, grad_out)
        return dx, doff, dw_, db, None, None, None


class ModDeformConvFunction(_DeformConvBase):
    """v2: mask is the already-activated modulation (2*sigmoid in ModDeformConv.forward); backward kernels K4-K6."""

    @staticmethod
    def forward(ctx, x, offset, mask, weight, bias=None, stride=1, padding=0, dilation=1):
        return _DeformConvBase._forward(ctx, x, offset, mask, weight, bias, stride, padding, dilation)

    @staticmethod
    def backward(ctx, grad_out):
        dx, doff, dmask, dw_, db = _DeformConvBase._backward(ctx, grad_out)
        return dx, doff, dmask, dw_, db, None, None, None


class RoIAlignFunction(torch.autograd.Function):
    """functions/roialign.py:21-58: forward = upsnet_roi_align_forward (NCHW fp32), backward = upsnet_roi_align_backward."""

    @staticmethod
    def forward(ctx, features, rois, pooled_height, pooled_width, spatial_scale, sampling_ratio=2):
        from . import operators as ops
        ctx.save_for_backward(rois)
        ctx.cfg = (tuple(features.shape), int(pooled_height), int(pooled_width), float(spatial_scale), int(sampling_ratio))
        return ops.roi_align(features, rois, pooled_height, pooled_width, spatial_scale, sampling_ratio)

    @staticmethod
    def backward(ctx, grad_out):
        (rois,) = ctx.saved_tensors
        (B, Cc, H, W), ph, pw, scale, sr = ctx.cfg
        if rois.shape[0] == 0:          # an empty grad_out has no data pointer for the C ABI; nothing to scatter
            return torch.zeros((B, Cc, H, W), dtype=torch.float32, device=grad_out.device), None, None, None, None, None
        grad_out, rois = f32c(grad_out), f32c(rois)
        dfeat = torch.empty((B, Cc, H, W), dtype=torch.float32, device=grad_out.device)
        with torch.cuda.device(grad_out.device):
            check(lib().upsnet_roi_align_backward(ptr(grad_out), ptr(rois), rois.shape[0], B, Cc, H, W, ph, pw, sr, scale,
                                                  ptr(dfeat), stream_ptr(grad_out.device)), "roi_align_backward")
        return dfeat, None, None, None, None, None


class OffsetConvFunction(torch.autograd.Function):
    """The 3x3 / pad 1 offset (and mask) conv of DeformConvWithOffset / ModDeformConvWithOffsetMask: forward is the same
    ops.conv2d the no-grad path runs (so the offsets, and where the samples land, do not depend on requires_grad); backward
    is the library's fp32 conv gradients with TF32 off, plus the bias sum."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        from . import operators as ops
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        return ops.conv2d(x, weight, bias, 1, 1, 1, out_format="nchw")

    @staticmethod
    def backward(ctx, grad_out):
        x, weight = ctx.saved_tensors
        grad_out = grad_out.float()
        dx = dw_ = None
        with torch.backends.cudnn.flags(enabled=torch.backends.cudnn.enabled, benchmark=torch.backends.cudnn.benchmark,
                                        deterministic=torch.backends.cudnn.deterministic, allow_tf32=False):
            if ctx.needs_input_grad[0]:
                dx = torch.nn.grad.conv2d_input(x.shape, weight, grad_out, stride=1, padding=1)
            if ctx.needs_input_grad[1]:
                dw_ = torch.nn.grad.conv2d_weight(x, weight.shape, grad_out, stride=1, padding=1)
        db = grad_out.sum(dim=(0, 2, 3)) if ctx.has_bias and ctx.needs_input_grad[2] else None
        return dx, dw_, db


class FPNRoIAlignFunction(torch.autograd.Function):
    """FPNRoIAlign on fp32 features [P2..P5]: forward = upsnet_roi_align_fpn_forward, which also writes the level it chose
    for every roi; backward = upsnet_roi_align_backward once per level on the output gradient with the rows of the other
    levels zeroed.  The levels come from the forward kernel, never recomputed on the host: a rounding difference at a level
    boundary would send a roi's gradient to the wrong level."""

    @staticmethod
    def forward(ctx, rois, pooled_height, pooled_width, spatial_scales, sampling_ratio, *feats):
        from . import operators as ops
        out, levels = ops.fpn_roi_align(list(feats), rois, pooled_height, pooled_width, spatial_scales, sampling_ratio,
                                        layout="auto", return_levels=True)
        ctx.save_for_backward(rois, levels)
        ctx.cfg = ([tuple(f.shape) for f in feats], int(pooled_height), int(pooled_width),
                   [float(s) for s in spatial_scales], int(sampling_ratio))
        return out

    @staticmethod
    def backward(ctx, grad_out):
        rois, levels = ctx.saved_tensors
        shapes, ph, pw, scales, sr = ctx.cfg
        grad_out, rois = f32c(grad_out), f32c(rois)
        R = rois.shape[0]
        dfeats = []
        with torch.cuda.device(grad_out.device):
            for lv, (B, Cc, H, W) in enumerate(shapes):
                if not ctx.needs_input_grad[5 + lv]:
                    dfeats.append(None)
                    continue
                if R == 0:
                    dfeats.append(torch.zeros((B, Cc, H, W), dtype=torch.float32, device=grad_out.device))
                    continue
                g = torch.where((levels == lv).view(R, 1, 1, 1), grad_out, 0.0).contiguous()
                dfeat = torch.empty((B, Cc, H, W), dtype=torch.float32, device=grad_out.device)
                check(lib().upsnet_roi_align_backward(ptr(g), ptr(rois), R, B, Cc, H, W, ph, pw, sr, scales[lv],
                                                      ptr(dfeat), stream_ptr(grad_out.device)), "roi_align_backward")
                dfeats.append(dfeat)
        return (None, None, None, None, None) + tuple(dfeats)


# ------------------------------------------------------------------------------------------------
# gradient all-reduce (config #4: "bf16, NCCL allreduce")
# ------------------------------------------------------------------------------------------------
class FlatBucketAllReduce:
    """Averages the gradients of `params` over the process group through flat buckets.

    * buckets are filled in REVERSE parameter order (the order backward produces gradients), `bucket_bytes` each;
    * `reduce_dtype` (bf16 on the NCCL path: half the interconnect bytes; the accumulation of 8 ranks in bf16 costs ~3 bits, the
      configuration BASELINE.json names) -- gradients are packed with a cast, reduced with SUM, and unpacked with 1/world;
    * `start()` launches every bucket's all_reduce asynchronously (NCCL: on its own stream, overlapping the optimiser's
      host work and, when called from autograd hooks, the rest of backward); `finish()` waits and writes p.grad back.
    No data-path collective exists at inference (DESIGN.md section 6); this is the one real exchange step of the path."""

    def __init__(self, params, bucket_bytes=25 << 20, reduce_dtype=torch.bfloat16, group=None):
        self.params = [p for p in params if p.requires_grad]
        self.group, self.dtype = group, reduce_dtype
        esize = torch.empty((), dtype=reduce_dtype).element_size()
        self.buckets, cur, cur_n = [], [], 0
        for p in reversed(self.params):
            cur.append(p); cur_n += p.numel()
            if cur_n * esize >= bucket_bytes:
                self.buckets.append(cur); cur, cur_n = [], 0
        if cur:
            self.buckets.append(cur)
        self._flat, self._work = [None] * len(self.buckets), []

    def start(self):
        assert dist.is_available() and dist.is_initialized()
        self._work = []
        for bi, bucket in enumerate(self.buckets):
            grads = [(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) for p in bucket]
            flat = torch.cat([g.to(self.dtype) for g in grads])
            self._flat[bi] = flat
            self._work.append(dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=self.group, async_op=True))
        return self

    def finish(self):
        world = dist.get_world_size(self.group)
        for bi, bucket in enumerate(self.buckets):
            self._work[bi].wait()
            flat, off = self._flat[bi], 0
            for p in bucket:
                n = p.numel()
                g = (flat[off:off + n].to(p.dtype) / world).view_as(p)
                if p.grad is None:
                    p.grad = g.clone()
                else:
                    p.grad.copy_(g)
                off += n
        self._work = []
        return self

    def __call__(self):
        return self.start().finish()


# ------------------------------------------------------------------------------------------------
# RPN training targets
# ------------------------------------------------------------------------------------------------
class RPNTargets:
    """add_rpn_blobs for one image on the device.

    Built from the reference's `config` (network.rpn_feat_stride, anchor_scales[0], anchor_ratios, rcnn_feat_stride;
    train.max_size, rpn_batch_size, rpn_fg_fraction, rpn_positive_overlap, rpn_negative_overlap, rpn_straddle_thresh) or
    from the same values as keywords.  Labels, weights and the dx / dy targets are bit-exact to the reference; dw / dh go
    through a float32 log (numpy's is not correctly rounded either).  The two np.random.choice draws are replaced by a
    seeded rule (include/upsnet_b200.h, upsnet_rpn_targets): the same seed gives the same targets."""

    def __init__(self, config=None, *, feat_strides=(4, 8, 16, 32, 64), anchor_scale=8, anchor_ratios=(0.5, 1, 2),
                 rcnn_feat_stride=32, max_size=1333, batch_size=256, fg_fraction=0.5, positive_overlap=0.7,
                 negative_overlap=0.3, straddle_thresh=0):
        from .detection import generate_anchors
        if config is not None:
            net, tr = config.network, config.train
            feat_strides, anchor_scale, anchor_ratios = net.rpn_feat_stride, net.anchor_scales[0], net.anchor_ratios
            rcnn_feat_stride, max_size, batch_size = net.rcnn_feat_stride, tr.max_size, tr.rpn_batch_size
            fg_fraction, positive_overlap = tr.rpn_fg_fraction, tr.rpn_positive_overlap
            negative_overlap, straddle_thresh = tr.rpn_negative_overlap, tr.rpn_straddle_thresh
        self.strides = [int(s) for s in feat_strides]
        fpn_max = rcnn_feat_stride * np.ceil(max_size / float(rcnn_feat_stride))          # generate_anchors.py:98-101
        self.field_sizes = [int(np.ceil(fpn_max / float(s))) for s in self.strides]
        self.cell = np.stack([generate_anchors(s, (anchor_scale * s,), anchor_ratios) for s in self.strides])
        self.A = self.cell.shape[1]
        self.num_anchors = sum(self.A * F * F for F in self.field_sizes)
        self.batch_size, self.num_fg = int(batch_size), int(fg_fraction * batch_size)   # assign_anchor.py:502
        self.pos, self.neg, self.straddle = float(positive_overlap), float(negative_overlap), float(straddle_thresh)
        self._dev = {}
        self.counts = None

    def _buffers(self, dev):
        if dev not in self._dev:
            sz = C.c_size_t()
            check(lib().upsnet_rpn_targets_workspace_bytes(self.num_anchors, self.batch_size, C.byref(sz)),
                  "rpn_targets_workspace_bytes")
            self._dev[dev] = (torch.from_numpy(np.ascontiguousarray(self.cell, np.float64)).to(dev),
                              torch.empty(sz.value, dtype=torch.uint8, device=dev))
        return self._dev[dev]

    def __call__(self, gt_boxes, im_height, im_width, seed=None):
        """gt_boxes: CUDA float32 [G,4] (already scaled); -> {'rpn_labels_fpn{s}': int64 [1,A,F,F],
        'rpn_bbox_targets_fpn{s}' / 'rpn_bbox_inside_weights_fpn{s}' / 'rpn_bbox_outside_weights_fpn{s}': float32
        [1,4A,F,F]} as views of four flat device tensors.  self.counts: int32 [4] on the device (inside anchors, fg
        candidates, final fg, final bg).  seed=None draws one from np.random, so np.random.seed governs it."""
        require_cuda(gt_boxes)
        gt = f32c(gt_boxes).reshape(-1, 4)
        if gt.shape[0] == 0:
            # the reference raises NameError here (anchor_to_gt_max is unbound without boxes)
            raise _lib.UpsnetError("rpn_targets: no ground-truth boxes")
        if seed is None:
            seed = int(np.random.randint(np.iinfo(np.int64).max, dtype=np.int64))
        dev = gt.device
        cell, ws = self._buffers(dev)
        N = self.num_anchors
        labels = torch.empty(N, dtype=torch.int64, device=dev)
        targets, inside, outside = (torch.empty(4 * N, dtype=torch.float32, device=dev) for _ in range(3))
        counts = torch.empty(4, dtype=torch.int32, device=dev)
        L = len(self.strides)
        with torch.cuda.device(dev):
            check(lib().upsnet_rpn_targets(ptr(gt), gt.shape[0], ptr(cell), (C.c_int * L)(*self.strides),
                                           (C.c_int * L)(*self.field_sizes), L, self.A, float(im_height),
                                           float(im_width), self.straddle, self.pos, self.neg, self.batch_size,
                                           self.num_fg, int(seed) & 0xFFFFFFFFFFFFFFFF, ptr(labels), ptr(targets),
                                           ptr(inside), ptr(outside), ptr(counts), ptr(ws), ws.numel(),
                                           stream_ptr(dev)), "rpn_targets")
        self.counts = counts
        out, off = {}, 0
        for s, F in zip(self.strides, self.field_sizes):
            n = self.A * F * F
            out["rpn_labels_fpn%d" % s] = labels[off:off + n].view(1, self.A, F, F)
            for name, t in (("rpn_bbox_targets_fpn%d", targets), ("rpn_bbox_inside_weights_fpn%d", inside),
                            ("rpn_bbox_outside_weights_fpn%d", outside)):
                out[name % s] = t[4 * off:4 * (off + n)].view(1, 4 * self.A, F, F)
            off += n
        return out

    def from_roidb(self, entry, im_scale, device, seed=None):
        """Drop-in for add_rpn_blobs on one roidb entry: boxes of a class > 0 that are not crowd, times the Python float
        im_scale (im_scales[0] of get_image_blob, assign_anchor.py:399); image size np.round(h * scale) (:391-392)."""
        keep = np.where((entry["gt_classes"] > 0) & (entry["is_crowd"] == 0))[0]
        boxes = (entry["boxes"][keep, :] * float(im_scale)).astype(np.float32)
        if boxes.shape[0] == 0:
            raise _lib.UpsnetError("rpn_targets: no ground-truth boxes")
        im_height = np.round(entry["height"] * im_scale)
        im_width = np.round(entry["width"] * im_scale)
        gt = torch.from_numpy(np.ascontiguousarray(boxes)).to(device)
        return self(gt, im_height, im_width, seed)


# ------------------------------------------------------------------------------------------------
# Mask R-CNN proposal targets
# ------------------------------------------------------------------------------------------------
class PackedGT:
    """The ground truth of one roidb entry on the device (ProposalTargets.pack_roidb): views of one int32 upload."""

    def __init__(self, buf, parts, G, O):
        self.buf, self.G, self.O = buf, G, O
        for name, (off, n, dtype) in parts.items():
            v = buf[off:off + n]
            setattr(self, name, v.view(torch.float32) if dtype == np.float32 else v)


class ProposalTargets:
    """ProposalMaskTarget.forward for one image on the device.

    Built from the reference's `config` (dataset.num_classes, train.batch_rois / fg_fraction / fg_thresh / bg_thresh_hi
    / bg_thresh_lo, network.bbox_reg_weights / mask_size / cls_agnostic_bbox_reg) or from the same values as keywords.
    Every output is bit-exact to the reference except the dw / dh targets, which go through a float32 log (numpy's is
    not correctly rounded either).  The two np.random.choice draws of sample_rois are replaced by the seeded rule of
    RPNTargets (include/upsnet_b200.h, upsnet_proposal_targets): the same seed gives the same targets.

    Unlike the reference, the proposals are not appended to the roidb entry: nothing downstream reads them
    (get_gt_rois keeps the rows of class > 0 only)."""

    def __init__(self, config=None, *, num_classes=81, batch_rois=512, fg_fraction=0.25, fg_thresh=0.5, bg_thresh_hi=0.5,
                 bg_thresh_lo=0.0, bbox_reg_weights=(10., 10., 5., 5.), mask_size=28, cls_agnostic_bbox_reg=False):
        if config is not None:
            net, tr = config.network, config.train
            num_classes, batch_rois, fg_fraction = config.dataset.num_classes, tr.batch_rois, tr.fg_fraction
            fg_thresh, bg_thresh_hi, bg_thresh_lo = tr.fg_thresh, tr.bg_thresh_hi, tr.bg_thresh_lo
            bbox_reg_weights, mask_size = net.bbox_reg_weights, net.mask_size
            cls_agnostic_bbox_reg = net.cls_agnostic_bbox_reg
        self.K, self.batch_rois, self.M = int(num_classes), int(batch_rois), int(mask_size)
        self.fg_per_image = int(np.round(fg_fraction * self.batch_rois))           # sample_rois.py:56 (half to even)
        self.fg_thresh, self.bg_hi, self.bg_lo = float(fg_thresh), float(bg_thresh_hi), float(bg_thresh_lo)
        self.weights = tuple(float(w) for w in bbox_reg_weights)
        self.cls_agnostic = bool(cls_agnostic_bbox_reg)
        self.mask_capacity = max(self.fg_per_image, 1)
        self.counts = None

    def pack_roidb(self, entry, device):
        """One host-to-device upload of the entry's ground truth: boxes, gt_classes, gt_overlaps' max / argmax,
        box_to_gt_ind_map and the float32 polygons of the non-crowd objects of class > 0."""
        boxes = np.ascontiguousarray(entry["boxes"], np.float32).reshape(-1, 4)
        G = boxes.shape[0]
        cls = np.asarray(entry["gt_classes"]).astype(np.int64)
        crowd = np.asarray(entry["is_crowd"]).astype(bool)
        if G == 0 or (cls <= 0).any():
            raise _lib.UpsnetError("proposal_targets: every gt row needs a class > 0 (json_dataset writes no other)")
        if (cls >= self.K).any():
            raise _lib.UpsnetError("proposal_targets: a gt class is not below num_classes")
        ov = entry["gt_overlaps"]
        ov = ov.toarray() if hasattr(ov, "toarray") else np.asarray(ov)
        b2g = np.asarray(entry["box_to_gt_ind_map"]).astype(np.int64)
        if ((b2g < -G) | (b2g >= G)).any():
            raise _lib.UpsnetError("proposal_targets: box_to_gt_ind_map out of range")
        obj = np.flatnonzero((cls > 0) & ~crowd)
        if obj.size == 0:
            # add_rpn_blobs fails on such an image in the reference, and RPNTargets.from_roidb raises there too
            raise _lib.UpsnetError("proposal_targets: no non-crowd ground truth")
        obj_boxes, obj_off, poly_off, verts = [], [0], [0], []
        for i in obj:
            segm = entry["segms"][i]
            if not isinstance(segm, list) or not segm:
                raise _lib.UpsnetError("proposal_targets: segmentation %d is not a polygon list" % i)
            ps = [np.asarray(p, np.float32) for p in segm]
            if any(p.ndim != 1 or p.size < 6 or p.size % 2 for p in ps):
                raise _lib.UpsnetError("proposal_targets: polygon of segmentation %d has an odd or < 6 coordinates" % i)
            allp = np.concatenate(ps)
            obj_boxes.append([allp[0::2].min(), allp[1::2].min(), allp[0::2].max(), allp[1::2].max()])
            for p in ps:
                verts.append(p)
                poly_off.append(poly_off[-1] + p.size // 2)
            obj_off.append(obj_off[-1] + len(ps))
        f32 = np.float32
        arrays = [("boxes", boxes.ravel(), f32), ("gt_max", ov.max(1).astype(f32), f32),
                  ("gt_maxcls", ov.argmax(1).astype(np.int32), np.int32), ("gt_classes", cls.astype(np.int32), np.int32),
                  ("gt_map", b2g.astype(np.int32), np.int32),
                  ("obj_boxes", np.asarray(obj_boxes, f32).ravel(), f32),
                  ("obj_poly", np.asarray(obj_off, np.int32), np.int32),
                  ("poly_vert", np.asarray(poly_off, np.int32), np.int32),
                  ("verts", np.concatenate(verts).astype(f32), f32)]
        parts, chunks, off = {}, [], 0
        for name, a, dt in arrays:
            a = np.ascontiguousarray(a, dt)
            parts[name] = (off, a.size, dt)
            chunks.append(a.view(np.int32))
            pad = (-a.size) % 4                     # 16-byte aligned parts
            chunks.append(np.zeros(pad, np.int32))
            off += a.size + pad
        buf = torch.from_numpy(np.concatenate(chunks)).to(device)
        return PackedGT(buf, parts, G, len(obj))

    def __call__(self, rois, packed, im_scale, seed=None):
        """rois: CUDA float32 [R,5]; packed: pack_roidb's; im_scale: the image's scale (float32).  -> dict of padded
        device buffers: rois [B,5], labels int64 [B], bbox_targets / bbox_inside_weights / bbox_outside_weights [B,4K],
        nongt_inds int64 [B] (-1 past its count), roi_has_mask uint8 [B], mask_rois [C,5], mask_int32 float32
        [C, K*M*M], with B = batch_rois and C = max(round(fg_fraction * B), 1).  self.counts: int32 [5] on the device
        (fg rows, bg rows, mask rows, error, nongt_inds count).  seed=None draws one from np.random."""
        require_cuda(rois)
        rois = f32c(rois).reshape(-1, 5)
        if seed is None:
            seed = int(np.random.randint(np.iinfo(np.int64).max, dtype=np.int64))
        dev = rois.device
        R, B, K, M, C_ = rois.shape[0], self.batch_rois, self.K, self.M, self.mask_capacity
        sz = C.c_size_t()
        check(lib().upsnet_proposal_targets_workspace_bytes(R, packed.G, B, C.byref(sz)),
              "proposal_targets_workspace_bytes")
        ws = torch.empty(sz.value, dtype=torch.uint8, device=dev)
        f = dict(device=dev, dtype=torch.float32)
        out = dict(rois=torch.empty((B, 5), **f), labels=torch.empty(B, dtype=torch.int64, device=dev),
                   bbox_targets=torch.empty((B, 4 * K), **f), bbox_inside_weights=torch.empty((B, 4 * K), **f),
                   bbox_outside_weights=torch.empty((B, 4 * K), **f), mask_rois=torch.empty((C_, 5), **f),
                   mask_int32=torch.empty((C_, K * M * M), **f),
                   roi_has_mask=torch.empty(B, dtype=torch.uint8, device=dev),
                   nongt_inds=torch.empty(B, dtype=torch.int64, device=dev))
        counts = torch.empty(5, dtype=torch.int32, device=dev)
        pk = packed
        with torch.cuda.device(dev):
            check(lib().upsnet_proposal_targets(
                ptr(rois) if R else None, R, ptr(pk.boxes), ptr(pk.gt_max), ptr(pk.gt_maxcls), ptr(pk.gt_classes),
                ptr(pk.gt_map), pk.G, ptr(pk.obj_boxes), ptr(pk.obj_poly), ptr(pk.poly_vert), ptr(pk.verts), pk.O,
                float(np.float32(im_scale)), K, B, self.fg_per_image, self.fg_thresh, self.bg_hi, self.bg_lo,
                *self.weights, int(self.cls_agnostic), M, int(seed) & 0xFFFFFFFFFFFFFFFF, ptr(out["rois"]),
                ptr(out["labels"]), ptr(out["bbox_targets"]), ptr(out["bbox_inside_weights"]),
                ptr(out["bbox_outside_weights"]), ptr(out["nongt_inds"]), ptr(out["mask_rois"]),
                ptr(out["mask_int32"]), ptr(out["roi_has_mask"]), ptr(counts), ptr(ws), ws.numel(),
                stream_ptr(dev)), "proposal_targets")
        self.counts = counts
        return out

    NAMES = ("rois", "labels", "bbox_targets", "bbox_inside_weights", "bbox_outside_weights", "mask_rois", "mask_int32",
             "roi_has_mask", "nongt_inds")

    def from_roidb(self, rois, entry, im_info, seed=None):
        """Drop-in for ProposalMaskTarget.forward(rois, roidb, im_info) on one image: its nine tensors (rois, labels
        int64, bbox_targets, the inside / outside weights, mask_rois, mask_int32 float32 [n_mask, K*M*M], roi_has_mask
        uint8, nongt_inds int64) as views of the device buffers.  One synchronisation, to read the counts."""
        im_scale = np.float32(np.asarray(im_info.cpu() if torch.is_tensor(im_info) else im_info).reshape(-1, 3)[0, 2])
        out = self(rois, self.pack_roidb(entry, rois.device), im_scale, seed)
        nf, nb, nm, err, nn = (int(v) for v in self.counts.cpu())
        if err:
            raise _lib.UpsnetError("proposal_targets: no fg and no bg rois (the reference raises IndexError)")
        n = nf + nb
        sl = dict(rois=n, labels=n, bbox_targets=n, bbox_inside_weights=n, bbox_outside_weights=n, mask_rois=nm,
                  mask_int32=nm, roi_has_mask=n, nongt_inds=nn)
        return tuple(out[k][:sl[k]] for k in self.NAMES)
