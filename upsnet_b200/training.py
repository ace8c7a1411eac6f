"""Training-side pieces of the hot path (BASELINE config #4: UPSNet-50 end2end_train, bf16, 8 GPUs, NCCL all-reduce):

* autograd Functions for the custom operators with hand-written sm_90a BACKWARD kernels (csrc/backward.cu):
    DeformConvFunction / ModDeformConvFunction   operators/functions/deform_conv.py:26-108, mod_deform_conv.py:25-118
    RoIAlignFunction                             operators/functions/roialign.py:21-58
    FPNRoIAlignFunction                          operators/modules/fpn_roi_align.py:32-62 (four RoIAlignFunction calls)
  The dense GEMMs of the deformable backward (d(weight) = dY col^T, d(col) = W^T dY) are library calls (torch.mm), like the
  reference's; the gather / scatter / coordinate-gradient kernels are ours.  OffsetConvFunction makes the offset conv of
  the *WithOffset* modules differentiable; its backward convs are library calls too.
* conv2d / linear / conv_transpose2x2 (Conv2dFunction, ConvTranspose2x2Function): the trainable dense convolutions and
  FC layers of models/{resnet,fpn,rpn,rcnn}.py with device gradients (csrc/conv_backward.cu).  Forward is ops.conv2d with
  the fused bias / residual / ReLU epilogue on the stored copy of x (hi/lo pair for bf16x3, bf16 NHWC for bf16), which
  is also all backward keeps of x; backward prepares g (ReLU mask, padded NHWC pair / bf16, d bias, d residual) in one
  pass, runs dX on the forward kernel with tap-flipped weights and dW on a split-K wgmma kernel, and launches only what
  needs_input_grad asks for.
* FlatBucketAllReduce: the gradient all-reduce of `upsnet_end2end_train.py:121` (hvd.DistributedOptimizer) as flat bf16
  buckets over torch.distributed (NCCL between the GPUs, gloo in the CPU tests): gradients are packed per bucket,
  reduced asynchronously while the rest of backward runs, averaged and unpacked before the optimiser step (or, with
  step(optimizer), packed on the device and applied by the optimiser straight from the reduced buckets).
* RPNTargets: the RPN training targets of one image (rpn/assign_anchor.py:370-595 add_rpn_blobs / _get_rpn_blobs, run by
  the reference's data loaders on the host) on the device (csrc/rpn_target.cu), as the label dict coco.py:133-142 builds.
* ProposalTargets: the Mask R-CNN proposal targets of one image (operators/modules/proposal_mask_target.py, run by the
  reference on the host in the middle of the forward) on the device (csrc/proposal_target.cu): roi sampling, box
  targets and the class-specific polygon mask targets.
* PanopticLabels: the label maps of the semantic and panoptic heads (seg_gt, seg_gt_4x, mask_gt, seg_roi_gt), built by
  the reference's data loaders on the host, on the device (csrc/labels.cu), with Pillow's polygon fill restated.
* TrainingSample: the (data, label) pair of one roidb entry as the reference's loader and collate yield it (scale draw,
  horizontal flip, image blob, im_info, RPN targets, label maps), from the decoded uint8 image and label map.
* PanopticLoss: the panoptic head of the training forward (models/resnet_upsnet.py:144-179: SegTerm, MaskTerm, the void
  logits, MaskMatching, calc_panoptic_acc and the cross-entropy) as one fused loss with hand-written forward and
  backward kernels (csrc/panoptic_loss.cu), plus the two host helpers for the lines before it (gt_rois, draw_keep).
* SemanticLoss, FcnRoiLoss, RPNLoss, MaskRCNNLoss: the other losses of the training forward
  (models/resnet_upsnet.py:127-142) with hand-written forward and backward kernels (csrc/train_loss.cu).  SemanticLoss evaluates the x4 up-sampling of
  fcn_score inside the cross-entropy, so the [1,S,4h,4w] fcn_output (159 MB at 1024x2048, S 19), its log-softmax and
  its gradient are never built; RPNLoss covers the five FPN levels in one launch and reads the label fields in place;
  MaskRCNNLoss reads mask_score and mask_target once.  FcnRoiLoss samples fcn_score where the reference samples the
  512-channel concat of the semantic head, so neither that concat nor the [R,512,28,28] roi features are built.
* SGD, LRSchedule: the optimiser (lib/nn/optimizer.py:19-106) with the learning-rate schedule and momentum decay of
  upsnet_end2end_train.py:76-103, 235-240, every parameter updated in one launch (csrc/sgd.cu), from p.grad or, through
  FlatBucketAllReduce.step, straight from the all-reduced bf16 buckets; with a schedule attached the step issues kernels
  only and can be replayed from a CUDA graph.  Unlike the reference, the step does not write g + wd p back into p.grad.
* FcnScoreFuseFunction / fcn_score_fuse_backward: the semantic head's level sum s2 + up2(s3) + up4(s4) + up8(s5) with
  its adjoint on the device (csrc/pool.cu upsnet_fcn_score_fuse_backward), used by the model's training forward.

Scope note: this is the operator / communication layer of the training configuration, the RPN and proposal targets,
the label maps, every loss of the training forward, the dense convolutions and FC layers with their gradients, and the
optimiser; resnet_upsnet.forward(data, label) (model.py) composes them into the training step of the Cityscapes
configuration and of the COCO configurations (network.fpn_with_gap, train.fcn_with_roi_loss through FcnRoiLoss).  Adam
and clip_grad (imported by the training script, never called) are not built.  The offset convs of the *WithOffset* modules (OffsetConvFunction) and the GEMMs of the deformable backward
stay library calls.
"""
import ctypes as C

import numpy as np
import torch
import torch.distributed as dist
from torch.nn.modules.utils import _pair
from torch.optim.optimizer import required

from . import _lib
from ._lib import call, f32c, query_bytes, require_cuda
from .geometry import prep_scale
from .operators import _weight_cache, prep_image


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
        for n in range(N):          # the reference loops over the batch as well (functions/deform_conv.py:84-104)
            m_n = None if mask is None else mask[n]
            go = grad_out[n].reshape(Cout, P)
            call("dcn_im2col", dev, x[n], offset[n], m_n, *g, col)
            dw_.addmm_(go, col.t())                                         # d(weight) += dY col^T
            dcol = torch.mm(w2.t(), go)                                     # d(col) = W^T dY
            call("dcn_col2im", dev, dcol, offset[n], m_n, *g, dx[n])
            call("dcn_col2im_coord", dev, dcol, x[n], offset[n], m_n, *g, doff[n], None if dmask is None else dmask[n])
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
        call("roi_align_backward", grad_out.device, grad_out, rois, rois.shape[0], B, Cc, H, W, ph, pw, sr, scale, dfeat)
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
        for lv, (B, Cc, H, W) in enumerate(shapes):
            if not ctx.needs_input_grad[5 + lv]:
                dfeats.append(None)
                continue
            if R == 0:
                dfeats.append(torch.zeros((B, Cc, H, W), dtype=torch.float32, device=grad_out.device))
                continue
            g = torch.where((levels == lv).view(R, 1, 1, 1), grad_out, 0.0).contiguous()
            dfeat = torch.empty((B, Cc, H, W), dtype=torch.float32, device=grad_out.device)
            call("roi_align_backward", grad_out.device, g, rois, R, B, Cc, H, W, ph, pw, sr, scales[lv], dfeat)
            dfeats.append(dfeat)
        return (None, None, None, None, None) + tuple(dfeats)


# ------------------------------------------------------------------------------------------------
# dense convolutions and FC layers with device gradients (csrc/conv_backward.cu)
# ------------------------------------------------------------------------------------------------
_CONV_PREC = {"bf16x3": _lib.PREC_BF16X3, "bf16": _lib.PREC_BF16}
_dgrad_cache = _weight_cache()


def _conv_prec(precision):
    if precision not in _CONV_PREC:
        raise ValueError("precision must be 'bf16x3' or 'bf16', got %r" % (precision,))
    return _CONV_PREC[precision]


def _stored_input(x, prec):
    """The copy of x the forward kernel reads, and the weight gradient reads again: the hi/lo pair store [N,H,W,2C]
    (bf16x3; the same bytes as the fp32 x) or bf16 NHWC [N,H,W,C] (bf16)."""
    from . import operators as ops
    x = x.detach()
    if prec == _lib.PREC_BF16X3:
        return ops.Pair.from_float(x).store
    return ops._nhwc(x.to(torch.bfloat16))


def _kernel_input(store, prec):
    """The stored copy as ops.conv2d takes it: a Pair, or the logical [N,C,H,W] bf16 view of the NHWC store."""
    from . import operators as ops
    return ops.Pair(store) if prec == _lib.PREC_BF16X3 else store.permute(0, 3, 1, 2)


def _check_conv_grad(N, Cin, H, W, weight, stride, padding, dilation, prec):
    """Raises UpsnetError, before any launch, for a layer whose backward the kernels do not cover: groups != 1, Cin % 64,
    stride > 1 with k > 1 or padding, a padding above d (k - 1) (no stride-1 data gradient as a convolution)."""
    Cout, Cin_w, kh, kw = weight.shape
    (sh, sw), (ph, pw), (dh, dw) = stride, padding, dilation
    if Cin_w != Cin:
        raise _lib.UpsnetError("conv2d backward: groups != 1 is not supported (weight %s, input channels %d)"
                               % (tuple(weight.shape), Cin))
    if (sh, sw) == (1, 1) and (ph > dh * (kh - 1) or pw > dw * (kw - 1)):
        raise _lib.UpsnetError("conv2d backward: padding %s above dilation * (k - 1)" % ((ph, pw),))
    query_bytes("conv_wgrad_workspace_bytes", N, H, W, Cin, Cout, kh, kw, sh, sw, ph, pw, dh, dw, prec)


def conv2d_backward(dy, x_store, y_store, weight, geom, prec, relu=False, has_bias=False, residual_up2=False,
                    need=(True, True, True, False), deconv=False):
    """Gradients of y = act(conv(x, W) + b [+ residual]) from dy (float32 logical [N,Cout,Ho,Wo], or [N,C,2Ho,2Wo] for
    the 2x2 deconv): (dx, dw, db, dres) for the four flags of `need`, None where not needed.  x_store: _stored_input(x);
    y_store: the forward's float32 NHWC output (read for the ReLU mask); geom: (N, Cin, H, W, stride, padding, dilation)
    of the forward.  dx and dres are float32 logical NCHW with channels_last storage.  Kernels only, no host sync:
    capturable in a CUDA graph."""
    from . import operators as ops
    need_x, need_w, need_b, need_r = need
    N, Cin, H, W, (sh, sw), (ph, pw), (dh, dw) = geom
    Cw, _, kh, kw = weight.shape           # deconv: the 1x1 weight [4 C, Cin, 1, 1]
    C = Cw // 4 if deconv else Cw
    dev = dy.device
    if dy.dtype != torch.float32:
        dy = dy.float()
    if dy.is_contiguous():
        nhwc = False
    elif dy.is_contiguous(memory_format=torch.channels_last):
        nhwc = True
    else:
        dy, nhwc = dy.contiguous(), False
    Ho, Wo = _conv_out(H, ph, dh, kh, sh), _conv_out(W, pw, dw, kw, sw)
    Cp = (Cw + 63) // 64 * 64
    pair = prec == _lib.PREC_BF16X3
    flags = ((_lib.GRAD_RELU if relu else 0) | (_lib.GRAD_RES_UP2 if residual_up2 and need_r else 0) |
             (_lib.GRAD_UNSHUFFLE2 if deconv else 0) | (_lib.GRAD_DY_NHWC if nhwc else 0))
    g = torch.empty((N, Ho, Wo, Cp * (2 if pair else 1)), dtype=torch.bfloat16, device=dev)
    db = torch.empty(C, dtype=torch.float32, device=dev) if (need_b and has_bias) else None
    dres = None
    if need_r:
        Hr, Wr = (Ho // 2, Wo // 2) if residual_up2 else (Ho, Wo)
        dres = torch.empty((N, Hr, Wr, C), dtype=torch.float32, device=dev)
    ws = None
    if db is not None:
        ws = torch.empty(query_bytes("conv_grad_prepare_workspace_bytes", N, C, Ho, Wo, flags), dtype=torch.uint8, device=dev)
    call("conv_grad_prepare", dev, dy, y_store if relu else None, g, db, dres, N, C, Ho, Wo, flags, prec,
         ws, 0 if ws is None else ws.numel())
    g_dt = _lib.DTYPE_PAIR if pair else _lib.DTYPE_BF16
    dx = dw_ = None
    if need_x:
        packed = ops._packed(_dgrad_cache, weight, "igemm_pack_weight_dgrad", "igemm_packed_weight_dgrad_bytes",
                             weight.shape)
        strided = (sh, sw) != (1, 1)
        qh, qw = (0, 0) if strided else (dh * (kh - 1) - ph, dw * (kw - 1) - pw)
        out = torch.empty((N, Ho, Wo, Cin) if strided else (N, H, W, Cin), dtype=torch.float32, device=dev)
        call("igemm_forward", dev, g, None, None, packed, None, None, out, N, Ho, Wo, Cp, Cin, kh, kw, 1, 1, qh, qw,
             dh, dw, _lib.LAYOUT_NHWC, g_dt, _lib.DTYPE_F32, 0, prec, None)
        if strided:
            full = torch.empty((N, H, W, Cin), dtype=torch.float32, device=dev)
            call("conv_dgrad_scatter2", dev, out, full, N, H, W, Cin)
            out = full
        dx = out.permute(0, 3, 1, 2)
    if need_w:
        nb = query_bytes("conv_wgrad_workspace_bytes", N, H, W, Cin, Cw, kh, kw, sh, sw, ph, pw, dh, dw, prec)
        wws = torch.empty(nb, dtype=torch.uint8, device=dev)
        dw_ = torch.empty((Cin, C, 2, 2) if deconv else tuple(weight.shape), dtype=torch.float32, device=dev)
        call("conv_wgrad", dev, x_store, g, dw_, N, H, W, Cin, Cw, kh, kw, sh, sw, ph, pw, dh, dw,
             _lib.GRAD_UNSHUFFLE2 if deconv else 0, prec, wws, nb)
    return dx, dw_, db, (None if dres is None else dres.permute(0, 3, 1, 2))


class Conv2dFunction(torch.autograd.Function):
    """y = act(conv(x, W) + b [+ residual]) with device gradients.  Forward: ops.conv2d on the stored copy of x (hi/lo pair
    for bf16x3, bf16 NHWC for bf16) with the fused epilogue and a float32 output, the same bytes as ops.conv2d of that
    copy; the copy is what backward keeps of x.  Backward (conv2d_backward): only what needs_input_grad asks for."""

    @staticmethod
    def forward(ctx, x, weight, bias, residual, stride, padding, dilation, residual_up2, relu, precision):
        from . import operators as ops
        require_cuda(x, weight, bias, residual)
        prec = _conv_prec(precision)
        stride, padding, dilation = _pair(stride), _pair(padding), _pair(dilation)
        N, Cin, H, W = x.shape
        _check_conv_grad(N, Cin, H, W, weight, stride, padding, dilation, prec)
        xs = _stored_input(x, prec)
        # the weight itself, not a detached copy: its packed form is cached on the tensor and its version, so a
        # parameter used several times in a step (the RPN head on five levels) is packed once
        y = ops.conv2d(_kernel_input(xs, prec), weight, None if bias is None else bias.detach(),
                       stride, padding, dilation, None if residual is None else residual.detach(), relu, prec,
                       out_dtype=torch.float32, residual_up2=residual_up2)
        ctx.save_for_backward(xs, y if relu else None, weight)
        ctx.cfg = ((N, Cin, H, W, stride, padding, dilation), prec, relu, bias is not None, residual_up2)
        return y

    @staticmethod
    def backward(ctx, grad_out):
        xs, y, weight = ctx.saved_tensors
        geom, prec, relu, has_bias, residual_up2 = ctx.cfg
        ni = ctx.needs_input_grad
        y_store = None if y is None else y.permute(0, 2, 3, 1)
        dx, dw_, db, dres = conv2d_backward(grad_out, xs, y_store, weight, geom, prec, relu, has_bias, residual_up2,
                                            (ni[0], ni[1], ni[2], ni[3]))
        return dx, dw_, db, dres, None, None, None, None, None, None


def conv2d(x, weight, bias=None, stride=1, padding=0, dilation=1, residual=None, residual_up2=False, relu=False,
           precision="bf16x3"):
    """Differentiable dense conv (groups 1) with the fused bias / residual / ReLU epilogue of ops.conv2d and device
    gradients (Conv2dFunction).  x float32 [N,Cin,H,W] (Cin % 64 == 0); weight [Cout,Cin,kh,kw]; stride 2 only for 1x1
    / pad 0; residual [N,Cout,Ho,Wo], or [N,Cout,Ho/2,Wo/2] with residual_up2 (nearest 2x up-sampling).
    -> float32 [N,Cout,Ho,Wo], channels_last storage."""
    return Conv2dFunction.apply(x, weight, bias, residual, stride, padding, dilation, residual_up2, relu, precision)


def linear(x, weight, bias=None, relu=False, precision="bf16x3"):
    """Differentiable y = x @ weight.T + bias (+ ReLU) as ops.linear computes it: a 1x1 conv over R one-pixel images.
    x float32 [R, K] (K % 64 == 0), weight [Cout, K] -> float32 [R, Cout]."""
    R, K = x.shape
    y = conv2d(x.reshape(R, K, 1, 1), weight.reshape(weight.shape[0], K, 1, 1), bias, relu=relu, precision=precision)
    return y.reshape(R, weight.shape[0])


class GroupNormFunction(torch.autograd.Function):
    """y = act(GN(x) + shift + up2(residual)) (ops.group_norm on float32 NHWC) with device gradients
    (upsnet_group_norm_backward): dx, d weight, d bias, d shift (float32 [N, C], the per-image d bias) and d residual,
    only what needs_input_grad asks for."""

    @staticmethod
    def forward(ctx, x, weight, bias, shift, residual, groups, eps, relu):
        from . import operators as ops
        require_cuda(x, weight, bias, shift, residual)
        xs = ops._nhwc(x.detach().float())
        y, stats = ops.group_norm(xs.permute(0, 3, 1, 2), weight.detach(), bias.detach(), groups, eps, relu,
                                  None if residual is None else residual.detach().float(), residual is not None,
                                  None if shift is None else shift.detach(), return_stats=True)
        ctx.save_for_backward(xs, y if relu else None, stats, weight)
        ctx.cfg = (groups, relu, residual is not None)
        return y

    @staticmethod
    def backward(ctx, grad_out):
        from . import operators as ops
        xs, y, stats, weight = ctx.saved_tensors
        groups, relu, has_res = ctx.cfg
        ni = ctx.needs_input_grad
        N, H, W, C = xs.shape
        dev = xs.device
        dy = ops._nhwc(grad_out.float())
        dx = torch.empty_like(xs)
        dgamma = torch.empty(C, dtype=torch.float32, device=dev) if ni[1] else None
        dbeta = torch.empty(C, dtype=torch.float32, device=dev) if ni[2] else None
        dshift = torch.empty((N, C), dtype=torch.float32, device=dev) if ni[3] else None
        dres = torch.empty((N, H // 2, W // 2, C), dtype=torch.float32, device=dev) if (has_res and ni[4]) else None
        nb = query_bytes("group_norm_backward_workspace_bytes", N, C, H, W, groups)
        ws = torch.empty(nb, dtype=torch.uint8, device=dev)
        flags = (_lib.EPI_RELU if relu else 0) | (_lib.EPI_RES_UP2 if has_res else 0)
        call("group_norm_backward", dev, dy, xs, None if y is None else y.permute(0, 2, 3, 1), stats, weight.detach(),
             dx, dgamma, dbeta, dshift, dres, N, C, H, W, groups, flags, ws, nb)
        return (dx.permute(0, 3, 1, 2), dgamma, dbeta, dshift, None if dres is None else dres.permute(0, 3, 1, 2),
                None, None, None)


def group_norm(x, weight, bias, groups=32, eps=1e-5, relu=False, residual=None, shift=None):
    """Differentiable nn.GroupNorm(groups, C) with the fused epilogue of ops.group_norm: x float32 [N,C,H,W] (or [R,C],
    normalised as [R,C,1,1], RCNN fc6); residual [N,C,H/2,W/2] added after nearest 2x up-sampling; shift [N,C].
    -> float32 of x's logical shape, channels_last storage."""
    if x.dim() == 2:
        R, C = x.shape
        return GroupNormFunction.apply(x.reshape(R, C, 1, 1), weight, bias, shift, residual, groups, eps, relu).reshape(R, C)
    return GroupNormFunction.apply(x, weight, bias, shift, residual, groups, eps, relu)


class ConvTranspose2x2Function(torch.autograd.Function):
    """ConvTranspose2d(k = 2, s = 2) (+ ReLU) as the 1x1 conv to 4 C channels ordered (a, b, c) that the engine runs
    (MaskBranch.prepare), followed by the pixel shuffle.  Backward reads dY through the 2x2 pixel-unshuffle of
    upsnet_conv_grad_prepare and writes d weight straight in the [Cin, C, 2, 2] layout."""

    @staticmethod
    def forward(ctx, x, weight, bias, relu, precision):
        from . import operators as ops
        require_cuda(x, weight, bias)
        prec = _conv_prec(precision)
        N, Cin, H, W = x.shape
        C = weight.shape[1]
        w1 = weight.detach().permute(2, 3, 1, 0).reshape(4 * C, Cin, 1, 1).contiguous()
        b1 = None if bias is None else bias.detach().repeat(4).contiguous()
        _check_conv_grad(N, Cin, H, W, w1, (1, 1), (0, 0), (1, 1), prec)
        xs = _stored_input(x, prec)
        y1 = ops.conv2d(_kernel_input(xs, prec), w1, b1, relu=relu, precision=prec, out_dtype=torch.float32)
        store = y1.permute(0, 2, 3, 1)                                   # NHWC [N, H, W, (a, b, c)]
        y = store.reshape(N, H, W, 2, 2, C).permute(0, 5, 1, 3, 2, 4).reshape(N, C, 2 * H, 2 * W)
        ctx.save_for_backward(xs, store if relu else None, w1)
        ctx.cfg = ((N, Cin, H, W, (1, 1), (0, 0), (1, 1)), prec, relu, bias is not None)
        return y

    @staticmethod
    def backward(ctx, grad_out):
        xs, store, w1 = ctx.saved_tensors
        geom, prec, relu, has_bias = ctx.cfg
        ni = ctx.needs_input_grad
        dx, dw_, db, _ = conv2d_backward(grad_out, xs, store, w1, geom, prec, relu, has_bias, False,
                                         (ni[0], ni[1], ni[2], False), deconv=True)
        return dx, dw_, db, None, None


def conv_transpose2x2(x, weight, bias=None, stride=2, relu=False, precision="bf16x3"):
    """Differentiable ConvTranspose2d with kernel = stride = 2, padding 0 (models/rcnn.py's mask deconv), with the ReLU
    that follows it fused when relu=True.  x float32 [N,Cin,H,W] (Cin % 64 == 0), weight [Cin,C,2,2] ->
    float32 [N,C,2H,2W].  Any other kernel size or stride raises."""
    k = tuple(weight.shape[2:])
    if k != (2, 2) or _pair(stride) != (2, 2):
        raise _lib.UpsnetError("conv_transpose2x2: kernel %s / stride %s; only kernel = stride = 2" % (k, _pair(stride)))
    return ConvTranspose2x2Function.apply(x, weight, bias, relu, precision)


def fcn_score_fuse_backward(dscore):
    """(ds3, ds4, ds5) = (up2^T, up4^T, up8^T)(dscore) for dscore float32 [N,C,H,W], H % 8 == W % 8 == 0: the adjoint of
    ops.fcn_score_fuse in one launch (upsnet_fcn_score_fuse_backward)."""
    require_cuda(dscore)
    g = f32c(dscore)
    N, Cc, H, W = g.shape
    outs = [torch.empty((N, Cc, H >> l, W >> l), dtype=torch.float32, device=g.device) for l in (1, 2, 3)]
    call("fcn_score_fuse_backward", g.device, g, *outs, N * Cc, H, W)
    return tuple(outs)


class FcnScoreFuseFunction(torch.autograd.Function):
    """score = s2 + up2(s3) + up4(s4) + up8(s5) (bilinear, align_corners=False): forward ops.fcn_score_fuse, backward
    its adjoint (fcn_score_fuse_backward); d s2 is the incoming gradient itself."""

    @staticmethod
    def forward(ctx, s2, s3, s4, s5):
        from . import operators as ops
        return ops.fcn_score_fuse(s2.detach(), s3.detach(), s4.detach(), s5.detach())

    @staticmethod
    def backward(ctx, grad):
        g = f32c(grad)
        return (g,) + fcn_score_fuse_backward(g)


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
        self._fused = None      # step(): (optimizer, world, bf16 buffers, apply tables, pack tables)

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

    def step(self, optimizer, lr=None):
        """start(); finish(); optimizer.step(lr) without the passes in between: every bucket is packed on the device
        (upsnet_sgd_pack) into a persistent bf16 buffer, its all_reduce starts asynchronously, and as each completes the
        optimiser is applied straight from the reduced bucket (upsnet_sgd_apply, 1/world folded in).  The same bytes as
        the three calls, except that p.grad is not written.  As after finish(), every parameter takes part (a None
        gradient packs as zeros).  `lr` as optimizer.step takes it: a value, or None with a schedule attached.  The
        bucket parameters must be exactly the optimiser's; bf16 buckets only."""
        assert dist.is_available() and dist.is_initialized()
        if not isinstance(optimizer, SGD):
            raise _lib.UpsnetError("FlatBucketAllReduce.step: the optimiser must be upsnet_b200.SGD")
        if self.dtype != torch.bfloat16:
            raise _lib.UpsnetError("FlatBucketAllReduce.step: reduce_dtype must be torch.bfloat16")
        if {id(p) for p in self.params} != {id(p) for p in optimizer._params} or len(self.params) != len(optimizer._params):
            raise _lib.UpsnetError("FlatBucketAllReduce.step: the buckets' parameters are not the optimiser's")
        lr = optimizer._check_lr(lr)
        dev = optimizer._dev
        for p in self.params:               # every parameter is updated, so every buffer exists after this step
            optimizer._buffer(p, optimizer._group_of[p])
        world = dist.get_world_size(self.group)
        if self._fused is None or self._fused[0] is not optimizer or self._fused[1] != world:
            flats = [torch.empty(sum(p.numel() for p in b), dtype=torch.bfloat16, device=dev) for b in self.buckets]
            tables = [optimizer._bucket_table(b, f, world) for b, f in zip(self.buckets, flats)]
            self._fused = (optimizer, world, flats, tables, [None] * len(self.buckets))
        _, _, flats, tables, packs = self._fused
        work = []
        for bi, bucket in enumerate(self.buckets):
            key = tuple(p.grad.data_ptr() if p.grad is not None else 0 for p in bucket)
            if packs[bi] is None or packs[bi][0] != key:
                packs[bi] = (key,) + _pack_table(bucket, flats[bi], dev)
            call("sgd_pack", dev, packs[bi][1], packs[bi][2])
            work.append(dist.all_reduce(flats[bi], op=dist.ReduceOp.SUM, group=self.group, async_op=True))
        for bi in range(len(self.buckets)):
            work[bi].wait()
            optimizer._apply(tables[bi][0], tables[bi][1], lr)
            _bump_versions(self.buckets[bi])
        optimizer._advance()
        return self


# ------------------------------------------------------------------------------------------------
# optimiser (lib/nn/optimizer.py SGD + the learning-rate schedule and momentum decay of upsnet_end2end_train.py)
# ------------------------------------------------------------------------------------------------
_CHUNK = 8192       # UPSNET_SGD_CHUNK
_MAX_GROUPS = 16    # UPSNET_SGD_MAX_GROUPS
_GRAD_F32, _GRAD_BF16, _GRAD_NONE = 0, 1, 2
_CHUNK_DT = np.dtype([("param", "<u8"), ("buf", "<u8"), ("grad", "<u8"), ("n", "<i4"), ("group", "<i4"),
                      ("kind", "<i4"), ("inv_world", "<f4")])        # upsnet_sgd_chunk
_PACK_DT = np.dtype([("grad", "<u8"), ("out", "<u8"), ("n", "<i4"), ("reserved", "<i4")])    # upsnet_sgd_pack_chunk


def _upload_table(rows, dtype, dev):
    a = np.zeros(len(rows), dtype)
    for i, r in enumerate(rows):
        a[i] = r
    return torch.from_numpy(a.view(np.uint8)).to(dev), len(rows)


def _pack_table(bucket, flat, dev):
    """(device table, entries) of upsnet_sgd_pack for one bucket: each gradient's chunks at its offset in `flat`."""
    rows, off = [], 0
    for p in bucket:
        g = p.grad
        if g is not None:
            if g.dtype != torch.float32 or g.device != flat.device or not g.is_contiguous():
                raise _lib.UpsnetError("FlatBucketAllReduce.step: gradients must be contiguous float32 on the device")
        for s in range(0, p.numel(), _CHUNK):
            n = min(_CHUNK, p.numel() - s)
            rows.append((0 if g is None else g.data_ptr() + 4 * s, flat.data_ptr() + 2 * (off + s), n, 0))
        off += p.numel()
    return _upload_table(rows, _PACK_DT, dev)


def _bump_versions(params):
    """The kernels write the parameters in place through raw pointers; advance their version counters as an in-place torch
    op would, so that what is keyed on (tensor, version) -- the packed weights of ops, autograd's saved-tensor check --
    sees the update.  Host only; a step replayed from a CUDA graph does not run it."""
    for p in params:
        torch.autograd.graph.increment_version(p)


class LRSchedule:
    """The learning rate of iteration `it`, adjust_learning_rate / lr_factor / lr_poly of upsnet_end2end_train.py:76-103
    restated with the same Python float operations (bit-identical values):
      'step': base_lr * (0.1 ** number of decay iterations <= it), after a warm-up from base_lr / 10 that is linear in
              it / warmup_iteration;
      'poly': base_lr * (1 - it / max_iteration) ** 0.9, during warm-up the smaller of that and the linear warm-up.
    Built from the reference's `config` (train.lr_schedule, lr, max_iteration, decay_iteration, warmup_iteration,
    begin_iteration) or from the same values as keywords.  table() is the float64 table of [begin_iteration,
    max_iteration) and decay_flags() marks the iterations i after which the training loop decays the momentum buffers
    (i + 1 in decay_iteration, whatever the schedule); SGD.attach_schedule uploads both."""

    def __init__(self, config=None, *, lr_schedule="step", base_lr=None, max_iteration=None, decay_iteration=(),
                 warmup_iteration=0, begin_iteration=0):
        if config is not None:
            tr = config.train
            lr_schedule, base_lr, max_iteration = tr.lr_schedule, tr.lr, tr.max_iteration
            decay_iteration, warmup_iteration = tr.decay_iteration, tr.warmup_iteration
            begin_iteration = getattr(tr, "begin_iteration", 0)
        if lr_schedule not in ("step", "poly"):
            raise _lib.UpsnetError("LRSchedule: lr_schedule must be 'step' or 'poly', not %r" % (lr_schedule,))
        if base_lr is None or max_iteration is None:
            raise _lib.UpsnetError("LRSchedule: base_lr and max_iteration are required")
        self.lr_schedule, self.base_lr, self.max_iteration = lr_schedule, base_lr, int(max_iteration)
        self.decay_iteration = list(decay_iteration)
        self.warmup_iteration, self.begin_iteration = warmup_iteration, int(begin_iteration)
        if not 0 <= self.begin_iteration < self.max_iteration:
            raise _lib.UpsnetError("LRSchedule: begin_iteration must be in [0, max_iteration)")

    def _warmup(self, it):
        alpha = it / self.warmup_iteration
        return self.base_lr * (1 / 10.0 * (1 - alpha) + alpha)

    def __call__(self, it):
        if self.lr_schedule == "step":
            if it < self.warmup_iteration:
                return self._warmup(it)
            idx = len(self.decay_iteration)
            for i, d in enumerate(self.decay_iteration):
                if it < d:
                    idx = i
                    break
            return self.base_lr * (0.1 ** idx)
        poly = self.base_lr * ((1 - float(it) / self.max_iteration) ** (0.9))
        if it < self.warmup_iteration:
            return min(self._warmup(it), poly)
        return poly

    def table(self):
        return np.array([self(i) for i in range(self.begin_iteration, self.max_iteration)], np.float64)

    def decay_flags(self):
        decay = set(self.decay_iteration)
        return np.array([(i + 1) in decay for i in range(self.begin_iteration, self.max_iteration)], np.uint8)


class SGD(torch.optim.Optimizer):
    """Drop-in for lib.nn.optimizer.SGD (momentum SGD with per-group learning-rate multipliers: the reference passes
    lr=1 and get_params_lr()'s groups, 'lr' 1 or 2 and an optional 'weight_decay'), every parameter updated in one
    launch (upsnet_sgd_apply; the rounding of each element is in include/upsnet_b200.h).

    * step(lr) has the reference's signature.  A parameter whose p.grad is None is skipped entirely.  With momentum 0
      the reference applies p -= g + wd p and ignores lr; so does this.
    * The momentum buffers live in one flat float32 allocation (each segment 16-byte aligned); state[p]['momentum_buffer']
      is a view of it, created the first time p has a gradient, so state_dict() aliases the buffers and the reference's
      decay loop (optimizer.state_dict()['state'][k]['momentum_buffer'].div_(10)) acts on them.  state_dict() /
      load_state_dict() use the reference's format; load_state_dict copies into the flat buffer.
    * attach_schedule(LRSchedule) and step() with no argument: the learning rate and the momentum decay come from device
      tables at a device iteration counter, which the step advances; such a step issues kernels only and can be captured
      in a CUDA graph (after one eager step, which uploads the chunk table).
    * Unlike the reference, p.grad is not written: the reference leaves g + wd p in it, which nothing reads.
    * An eager step advances the version counter of every parameter, as an in-place torch op would; a step replayed
      from a CUDA graph cannot, so code that caches per (tensor, version) must be told (resnet_upsnet does this itself).
    * zero_grad() zeroes gradients in place (set_to_none=False, the reference's torch behaviour), so their pointers and
      the cached chunk table stay valid.  dampening != 0 raises, as the reference asserts; nesterov is not built.
    float32 CUDA parameters on one device only."""

    def __init__(self, params, lr=required, momentum=0, dampening=0, weight_decay=0,
                 nesterov=False):
        if nesterov:
            raise _lib.UpsnetError("SGD: nesterov momentum is not built")
        if dampening != 0:
            raise _lib.UpsnetError("SGD: dampening is not implemented (the reference asserts dampening == 0)")
        super().__init__(params, dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay,
                                      nesterov=nesterov))
        if any(g["nesterov"] for g in self.param_groups):
            raise _lib.UpsnetError("SGD: nesterov momentum is not built")
        if any(g["dampening"] != 0 for g in self.param_groups):
            raise _lib.UpsnetError("SGD: dampening is not implemented (the reference asserts dampening == 0)")
        if len(self.param_groups) > _MAX_GROUPS:
            raise _lib.UpsnetError("SGD: at most %d parameter groups" % _MAX_GROUPS)
        self._params = [p for g in self.param_groups for p in g["params"]]
        if not self._params:
            raise _lib.UpsnetError("SGD: no parameters")
        for p in self._params:
            if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous():
                raise _lib.UpsnetError("SGD: parameters must be contiguous float32 CUDA tensors, not %s %s"
                                       % (p.dtype, p.device))
        self._dev = self._params[0].device
        if any(p.device != self._dev for p in self._params):
            raise _lib.UpsnetError("SGD: every parameter must be on one device")
        offs, n = [], 0
        for p in self._params:
            offs.append(n)
            n += (p.numel() + 3) // 4 * 4
        self._flat = torch.zeros(max(n, 4), dtype=torch.float32, device=self._dev)
        self._views = {p: self._flat[o:o + p.numel()].view_as(p) for p, o in zip(self._params, offs)}
        self._group_of = {p: gi for gi, g in enumerate(self.param_groups) for p in g["params"]}
        self._table_key, self._table = None, None
        self._sched = None

    # -- the reference's interface --------------------------------------------------------------
    def zero_grad(self, set_to_none=False):
        super().zero_grad(set_to_none=set_to_none)

    def step(self, lr=None, closure=None):
        loss = closure() if closure is not None else None
        lr = self._check_lr(lr)
        key = tuple(p.grad.data_ptr() if p.grad is not None else 0 for p in self._params)
        if key != self._table_key:
            self._table, self._table_key = self._grad_table(), key
        self._apply(self._table[0], self._table[1], lr)
        _bump_versions(self._params)
        self._advance()
        return loss

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        loaded = {p: s["momentum_buffer"] for p, s in self.state.items() if "momentum_buffer" in s}
        self._flat.zero_()
        for p, v in self._views.items():
            if p in loaded:
                v.copy_(loaded[p])
                self.state[p]["momentum_buffer"] = v
        self._table_key = None

    # -- schedule ----------------------------------------------------------------------------------
    def attach_schedule(self, schedule):
        """Learning rate and momentum decay from `schedule` (an LRSchedule) on the device; the device iteration counter
        starts at schedule.begin_iteration.  step() then takes no argument."""
        if not isinstance(schedule, LRSchedule):
            raise _lib.UpsnetError("SGD.attach_schedule: an LRSchedule is required")
        self._sched = (schedule, torch.from_numpy(schedule.table()).to(self._dev),
                       torch.from_numpy(schedule.decay_flags()).to(self._dev),
                       torch.full((1,), schedule.begin_iteration, dtype=torch.int32, device=self._dev))

    @property
    def iteration(self):
        """The device iteration counter of the attached schedule (reads the device)."""
        return None if self._sched is None else int(self._sched[3].item())

    # -- internals ---------------------------------------------------------------------------------
    def _check_lr(self, lr):
        if self._sched is not None and lr is not None:
            raise _lib.UpsnetError("SGD.step: a schedule is attached; call step() without a learning rate")
        if self._sched is None and lr is None:
            raise _lib.UpsnetError("SGD.step: a learning rate is required (or attach_schedule first)")
        return None if lr is None else float(lr)

    def _buffer(self, p, gi):
        """The flat-buffer address of p's momentum buffer, created (as +0) on its first use; 0 without momentum."""
        if self.param_groups[gi]["momentum"] == 0:
            return 0
        st = self.state[p]
        if "momentum_buffer" not in st:
            self._views[p].zero_()
            st["momentum_buffer"] = self._views[p]
        return self._views[p].data_ptr()

    def _grad_table(self):
        rows = []
        for p in self._params:
            gi = self._group_of[p]
            g = p.grad
            if g is None:
                if p in self.state and "momentum_buffer" in self.state[p]:
                    kind, gp = _GRAD_NONE, 0
                else:
                    continue
            else:
                if g.dtype != torch.float32 or g.device != self._dev or not g.is_contiguous():
                    raise _lib.UpsnetError("SGD.step: gradients must be contiguous float32 on the parameters' device")
                kind, gp = _GRAD_F32, g.data_ptr()
            bp = self._buffer(p, gi)
            rows += self._rows(p, bp, gp, 4, gi, kind, 1.0)
        return _upload_table(rows, _CHUNK_DT, self._dev)

    def _bucket_table(self, bucket, flat, world):
        """The chunk table of one bf16 bucket (FlatBucketAllReduce.step): every parameter, gradient = its segment."""
        rows, off = [], 0
        inv = float(np.float32(1.0) / np.float32(world))
        for p in bucket:
            gi = self._group_of[p]
            rows += self._rows(p, self._buffer(p, gi), flat.data_ptr() + 2 * off, 2, gi, _GRAD_BF16, inv)
            off += p.numel()
        return _upload_table(rows, _CHUNK_DT, self._dev)

    @staticmethod
    def _rows(p, bp, gp, gsize, gi, kind, inv):
        rows = []
        for s in range(0, p.numel(), _CHUNK):
            rows.append((p.data_ptr() + 4 * s, bp + 4 * s if bp else 0, gp + gsize * s if gp else 0,
                         min(_CHUNK, p.numel() - s), gi, kind, inv))
        return rows

    def _apply(self, table, n, lr):
        groups = self.param_groups
        glr = (C.c_double * len(groups))(*[float(g["lr"]) for g in groups])
        wd = (C.c_float * len(groups))(*[float(g["weight_decay"]) for g in groups])
        mom = (C.c_float * len(groups))(*[float(g["momentum"]) for g in groups])
        if self._sched is None:
            call("sgd_apply", self._dev, table, n, len(groups), glr, wd, mom, lr, None, None, None, 0, 0)
        else:
            sch, lrt, dec, it = self._sched
            call("sgd_apply", self._dev, table, n, len(groups), glr, wd, mom, 0.0, lrt, dec, it, sch.begin_iteration,
                 lrt.numel())

    def _advance(self):
        if self._sched is not None:
            call("sgd_advance", self._dev, self._sched[3])


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
            sz = query_bytes("rpn_targets_workspace_bytes", self.num_anchors, self.batch_size)
            self._dev[dev] = (torch.from_numpy(np.ascontiguousarray(self.cell, np.float64)).to(dev),
                              torch.empty(sz, dtype=torch.uint8, device=dev))
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
        call("rpn_targets", dev, gt, gt.shape[0], cell, (C.c_int * L)(*self.strides),
             (C.c_int * L)(*self.field_sizes), L, self.A, float(im_height),
             float(im_width), self.straddle, self.pos, self.neg, self.batch_size,
             self.num_fg, int(seed) & 0xFFFFFFFFFFFFFFFF, labels, targets,
             inside, outside, counts, ws, ws.numel())
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
def pack_polygons(segms, rows, what):
    """The polygon layout shared by ProposalTargets.pack_roidb and PanopticLabels.pack_roidb: segms[i] for i in rows,
    each a non-empty list of flat [x0, y0, x1, y1, ...] polygons of >= 6 coordinates (dict / RLE segmentations are
    rejected).  -> (obj_poly int32 [n+1]: first polygon of each object, poly_vert int32 [P+1]: first vertex of each
    polygon, per object the list of its float64 polygons)."""
    obj_off, poly_off, polys = [0], [0], []
    for i in rows:
        segm = segms[i]
        if not isinstance(segm, list) or not segm:
            raise _lib.UpsnetError("%s: segmentation %d is not a polygon list" % (what, i))
        ps = [np.asarray(p, np.float64) for p in segm]
        if any(p.ndim != 1 or p.size < 6 or p.size % 2 for p in ps):
            raise _lib.UpsnetError("%s: polygon of segmentation %d has an odd or < 6 coordinates" % (what, i))
        for p in ps:
            poly_off.append(poly_off[-1] + p.size // 2)
        obj_off.append(obj_off[-1] + len(ps))
        polys.append(ps)
    return np.asarray(obj_off, np.int32), np.asarray(poly_off, np.int32), polys


def _upload_parts(arrays, device):
    """[(name, array, dtype)] -> (one int32 device buffer with every part 16-byte aligned, {name: (offset, size,
    dtype)})."""
    parts, chunks, off = {}, [], 0
    for name, a, dt in arrays:
        a = np.ascontiguousarray(a, dt)
        parts[name] = (off, a.size, dt)
        chunks.append(a.view(np.int32))
        pad = (-a.size) % 4
        chunks.append(np.zeros(pad, np.int32))
        off += a.size + pad
    return torch.from_numpy(np.concatenate(chunks)).to(device), parts


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
        obj_off, poly_off, polys = pack_polygons(entry["segms"], obj, "proposal_targets")
        obj_boxes, verts = [], []
        for ps in polys:
            ps = [p.astype(np.float32) for p in ps]
            allp = np.concatenate(ps)
            obj_boxes.append([allp[0::2].min(), allp[1::2].min(), allp[0::2].max(), allp[1::2].max()])
            verts.extend(ps)
        f32 = np.float32
        arrays = [("boxes", boxes.ravel(), f32), ("gt_max", ov.max(1).astype(f32), f32),
                  ("gt_maxcls", ov.argmax(1).astype(np.int32), np.int32), ("gt_classes", cls.astype(np.int32), np.int32),
                  ("gt_map", b2g.astype(np.int32), np.int32),
                  ("obj_boxes", np.asarray(obj_boxes, f32).ravel(), f32),
                  ("obj_poly", obj_off, np.int32), ("poly_vert", poly_off, np.int32),
                  ("verts", np.concatenate(verts).astype(f32), f32)]
        buf, parts = _upload_parts(arrays, device)
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
        sz = query_bytes("proposal_targets_workspace_bytes", R, packed.G, B)
        ws = torch.empty(sz, dtype=torch.uint8, device=dev)
        f = dict(device=dev, dtype=torch.float32)
        out = dict(rois=torch.empty((B, 5), **f), labels=torch.empty(B, dtype=torch.int64, device=dev),
                   bbox_targets=torch.empty((B, 4 * K), **f), bbox_inside_weights=torch.empty((B, 4 * K), **f),
                   bbox_outside_weights=torch.empty((B, 4 * K), **f), mask_rois=torch.empty((C_, 5), **f),
                   mask_int32=torch.empty((C_, K * M * M), **f),
                   roi_has_mask=torch.empty(B, dtype=torch.uint8, device=dev),
                   nongt_inds=torch.empty(B, dtype=torch.int64, device=dev))
        counts = torch.empty(5, dtype=torch.int32, device=dev)
        pk = packed
        call("proposal_targets", dev, rois if R else None, R, pk.boxes, pk.gt_max, pk.gt_maxcls, pk.gt_classes,
             pk.gt_map, pk.G, pk.obj_boxes, pk.obj_poly, pk.poly_vert, pk.verts, pk.O,
             float(np.float32(im_scale)), K, B, self.fg_per_image, self.fg_thresh, self.bg_hi, self.bg_lo,
             *self.weights, int(self.cls_agnostic), M, int(seed) & 0xFFFFFFFFFFFFFFFF, out["rois"],
             out["labels"], out["bbox_targets"], out["bbox_inside_weights"],
             out["bbox_outside_weights"], out["nongt_inds"], out["mask_rois"],
             out["mask_int32"], out["roi_has_mask"], counts, ws, ws.numel())
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


# ------------------------------------------------------------------------------------------------
# panoptic head loss
# ------------------------------------------------------------------------------------------------
_GAMMA = np.uint64(0x9E3779B97F4A7C15)


def _splitmix64(x):
    with np.errstate(over="ignore"):
        z = x + _GAMMA
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def draw_keys(seed, n):
    """uint64 [n]: the key of every candidate position of a draw, csrc/targets.cuh draw_key on stream 0."""
    with np.errstate(over="ignore"):
        return _splitmix64(np.uint64(int(seed) & 0xFFFFFFFFFFFFFFFF) ^ (np.arange(n, dtype=np.uint64) * _GAMMA))


def draw_keep(G, fraction, seed=None):
    """The keep_inds draw of models/resnet_upsnet.py:149, np.random.choice(G, max(int(G * fraction), 1), replace=False),
    by the seeded rule of the target classes: the positions with the smallest draw_keys(seed, G), in ascending key
    order (int64).  seed=None draws one from np.random, so np.random.seed governs it."""
    if G <= 0:
        raise _lib.UpsnetError("draw_keep: no ground-truth boxes")
    if seed is None:
        seed = int(np.random.randint(np.iinfo(np.int64).max, dtype=np.int64))
    size = max(int(G * fraction), 1)
    return np.argsort(draw_keys(seed, G), kind="stable")[:size].astype(np.int64)


def gt_rois(entry, im_scale, device):
    """get_gt_rois (models/resnet_upsnet.py:287-291) of one roidb entry: the non-crowd boxes of a class > 0 times the
    float32 im_scale (im_info[0, 2]) as float32 [n,5] rows (0, x1, y1, x2, y2), and their classes (int64 [n]), on
    `device`."""
    inds = np.where((entry["gt_classes"] > 0) & (entry["is_crowd"] == 0))[0]
    boxes = (np.asarray(entry["boxes"], np.float32)[inds] * np.float32(im_scale)).astype(np.float32)
    rois = np.hstack((np.zeros((boxes.shape[0], 1), np.float32), boxes.reshape(-1, 4)))
    cls = np.asarray(entry["gt_classes"])[inds].astype(np.int64)
    return torch.from_numpy(rois).to(device), torch.from_numpy(cls).to(device)


def _pl_workspace(k, h, w, dev):
    sz = query_bytes("panoptic_loss_workspace_bytes", k, h, w)
    return torch.empty(sz, dtype=torch.uint8, device=dev)


class PanopticLossFunction(torch.autograd.Function):
    """(loss, accuracy, counts) = the fused panoptic loss (include/upsnet_b200.h, upsnet_panoptic_loss_forward);
    differentiable in fcn_score and mask_score.  Inputs are validated by PanopticLoss.forward."""

    @staticmethod
    def forward(ctx, fcn_score, mask_score, gt_rois, cls_idx, seg_gt, mask_gt, keep_inds, num_classes, enable_void,
                box_scale, mask_size):
        dev = fcn_score.device
        _, S, h, w = fcn_score.shape
        k, Cm = mask_score.shape[0], mask_score.shape[1]
        fcn, msk = f32c(fcn_score.detach()), f32c(mask_score.detach())
        loss, acc = (torch.empty((), dtype=torch.float32, device=dev) for _ in range(2))
        counts = torch.empty(2, dtype=torch.int32, device=dev)
        lse = torch.empty(h * w, dtype=torch.float32, device=dev)
        gtc = torch.empty(h * w, dtype=torch.int32, device=dev)
        ws = _pl_workspace(k, h, w, dev)
        call("panoptic_loss_forward", dev, fcn, S, h, w, msk, k, Cm, mask_size, gt_rois, cls_idx, seg_gt, mask_gt,
             int(mask_gt.dtype == torch.int64), mask_gt.shape[0], keep_inds, num_classes, int(enable_void),
             box_scale, loss, acc, counts, lse, gtc, ws, ws.numel())
        ctx.save_for_backward(fcn, msk, gt_rois, cls_idx, lse, gtc)
        ctx.cfg = (num_classes, int(enable_void), box_scale, mask_size)
        ctx.mark_non_differentiable(acc, counts)
        return loss, acc, counts

    @staticmethod
    def backward(ctx, grad_loss, _grad_acc, _grad_counts):
        fcn, msk, rois, cls, lse, gtc = ctx.saved_tensors
        num_classes, enable_void, box_scale, mask_size = ctx.cfg
        dev = fcn.device
        _, S, h, w = fcn.shape
        k, Cm = msk.shape[0], msk.shape[1]
        go = f32c(grad_loss).reshape(1)
        dfcn = torch.empty_like(fcn) if ctx.needs_input_grad[0] else None
        dmsk = torch.empty_like(msk) if ctx.needs_input_grad[1] else None
        if dfcn is not None or dmsk is not None:
            ws = _pl_workspace(k, h, w, dev)
            call("panoptic_loss_backward", dev, fcn, S, h, w, msk, k, Cm, mask_size, rois, cls, num_classes, enable_void,
                 box_scale, lse, gtc, go, dfcn, dmsk, ws, ws.numel())
        return (dfcn, dmsk) + (None,) * 9


class PanopticLoss(torch.nn.Module):
    """The panoptic head of the training forward of one image (models/resnet_upsnet.py:156-179, 250-257) as one fused,
    parameter-free loss: the class gather of mask_score, SegTerm, MaskTerm, the void logits, MaskMatching, the
    cross-entropy (ignore 255, mean over all pixels) and calc_panoptic_acc, without building a [1,k,h,w] plane and
    without a host read.  Built from the reference's `config` (dataset.num_seg_classes / num_classes,
    network.mask_size, enable_void = train.panoptic_box_keep_fraction < 1) or from the same values as keywords.

    Ground-truth boxes are never negative; a negative SegTerm bound is clamped to 0 here, where the reference's Python
    slice would wrap around, so no parity is claimed for such boxes.  The same inputs give the same bytes."""

    def __init__(self, config=None, *, num_seg_classes=None, num_classes=None, enable_void=True, box_scale=1 / 4.0,
                 mask_size=28):
        super().__init__()
        if config is not None:
            num_seg_classes, num_classes = config.dataset.num_seg_classes, config.dataset.num_classes
            mask_size = config.network.mask_size
            enable_void = config.train.panoptic_box_keep_fraction < 1
        if num_seg_classes is None or num_classes is None:
            raise _lib.UpsnetError("panoptic_loss: num_seg_classes and num_classes are required")
        self.num_seg_classes, self.num_classes = int(num_seg_classes), int(num_classes)
        self.enable_void, self.box_scale, self.mask_size = bool(enable_void), float(box_scale), int(mask_size)
        self.counts = None

    @staticmethod
    def _labels(seg_gt_4x, mask_gt, keep_inds):
        """-> (seg int64 [1,h,w], mask_gt uint8 / int64 [G,h,w], keep_inds int64 on the device or None), checked."""
        require_cuda(seg_gt_4x, mask_gt)
        if seg_gt_4x.dim() != 3 or seg_gt_4x.shape[0] != 1:
            raise _lib.UpsnetError("panoptic_loss: seg_gt_4x must be [1,h,w] (one image)")
        if mask_gt.dim() != 3 or mask_gt.shape[0] == 0 or mask_gt.shape[1:] != seg_gt_4x.shape[1:]:
            raise _lib.UpsnetError("panoptic_loss: mask_gt must be [G,h,w] with G >= 1 and the size of seg_gt_4x")
        if mask_gt.dtype not in (torch.uint8, torch.int64):
            raise _lib.UpsnetError("panoptic_loss: mask_gt must be uint8 or int64")
        if keep_inds is not None:
            if not torch.is_tensor(keep_inds) or not keep_inds.is_cuda:
                host = np.asarray(keep_inds.cpu() if torch.is_tensor(keep_inds) else keep_inds).astype(np.int64).reshape(-1)
                if host.size == 0 or host.min() < 0 or host.max() >= mask_gt.shape[0]:
                    raise _lib.UpsnetError("panoptic_loss: keep_inds must index mask_gt")
                keep_inds = torch.from_numpy(host).to(mask_gt.device)
            keep_inds = keep_inds.to(torch.int64).reshape(-1).contiguous()
        return seg_gt_4x.to(torch.int64).contiguous(), mask_gt.contiguous(), keep_inds

    def panoptic_gt(self, seg_gt_4x, mask_gt, keep_inds=None):
        """MaskMatching.forward: the int64 [1,h,w] ground truth of the panoptic logits."""
        seg, mgt, keep = self._labels(seg_gt_4x, mask_gt, keep_inds)
        out = torch.empty_like(seg)
        _, h, w = seg.shape
        call("panoptic_gt", seg.device, seg, mgt, int(mgt.dtype == torch.int64), mgt.shape[0], keep,
             0 if keep is None else keep.numel(), h, w, self.num_seg_classes,
             self.num_classes, out)
        return out

    def forward(self, fcn_score, mask_score, gt_rois, cls_idx, seg_gt_4x, mask_gt, keep_inds=None):
        """fcn_score [1,S,h,w]; mask_score [k,C,M,M] with C = num_classes (the mask branch's output on gt_rois) or 1
        (already gathered); gt_rois [k,5] and cls_idx [k], after keep_inds when there is a draw; seg_gt_4x [1,h,w];
        mask_gt [G,h,w] uint8 or int64; keep_inds [k] (tensor or numpy) or None.  -> (loss, accuracy), 0-dim device
        tensors; self.counts: int32 [2] on the device (correct pixels, ignored pixels)."""
        E = _lib.UpsnetError
        require_cuda(fcn_score, mask_score, gt_rois, cls_idx)
        if self.enable_void != (keep_inds is not None):
            raise E("panoptic_loss: enable_void goes with keep_inds (the reference sets the two together)")
        if fcn_score.dim() != 4 or fcn_score.shape[0] != 1:
            raise E("panoptic_loss: only batch size 1 (fcn_score [1,S,h,w])")
        if fcn_score.shape[1] != self.num_seg_classes:
            raise E("panoptic_loss: fcn_score has %d channels, not num_seg_classes" % fcn_score.shape[1])
        k = mask_score.shape[0]
        if k == 0:
            raise E("panoptic_loss: no ground-truth boxes")
        M = self.mask_size
        if mask_score.dim() != 4 or mask_score.shape[1] not in (1, self.num_classes) or tuple(mask_score.shape[2:]) != (M, M):
            raise E("panoptic_loss: mask_score must be [k,num_classes,%d,%d] or [k,1,%d,%d]" % (M, M, M, M))
        if tuple(gt_rois.shape) != (k, 5) or cls_idx.numel() != k:
            raise E("panoptic_loss: gt_rois must be [k,5] and cls_idx [k], k = mask_score.shape[0]")
        seg, mgt, keep = self._labels(seg_gt_4x, mask_gt, keep_inds)
        if seg.shape[1:] != fcn_score.shape[2:]:
            raise E("panoptic_loss: seg_gt_4x and fcn_score differ in size")
        if (keep.numel() if keep is not None else mgt.shape[0]) != k:
            raise E("panoptic_loss: one ground-truth mask per box (keep_inds, or all of mask_gt, must have k entries)")
        loss, acc, counts = PanopticLossFunction.apply(
            fcn_score, mask_score, f32c(gt_rois), cls_idx.to(torch.int64).reshape(-1).contiguous(), seg, mgt, keep,
            self.num_classes, self.enable_void, self.box_scale, M)
        self.counts = counts
        return loss, acc


# ------------------------------------------------------------------------------------------------
# semantic, RPN and Mask R-CNN losses
# ------------------------------------------------------------------------------------------------
def _scalars(dev, n):
    return [torch.empty((), dtype=torch.float32, device=dev) for _ in range(n)]


def _grad(g, dev):
    """A loss's incoming gradient as a float32 [1] device tensor (zero when autograd passes None)."""
    return torch.zeros(1, dtype=torch.float32, device=dev) if g is None else f32c(g).reshape(1)


class SemanticLossFunction(torch.autograd.Function):
    """(loss, counts) = the fused semantic loss (include/upsnet_b200.h, upsnet_semantic_loss_forward); differentiable in
    fcn_score.  Inputs are validated by SemanticLoss.forward."""

    @staticmethod
    def forward(ctx, fcn_score, seg_gt):
        dev = fcn_score.device
        _, S, h, w = fcn_score.shape
        fcn = f32c(fcn_score.detach())
        (loss,) = _scalars(dev, 1)
        counts = torch.empty(2, dtype=torch.int32, device=dev)
        lse = torch.empty(16 * h * w, dtype=torch.float32, device=dev)
        ws = torch.empty(query_bytes("semantic_loss_workspace_bytes", h, w), dtype=torch.uint8, device=dev)
        is64 = int(seg_gt.dtype == torch.int64)
        call("semantic_loss_forward", dev, fcn, S, h, w, seg_gt, is64, loss, counts, lse, ws, ws.numel())
        ctx.save_for_backward(fcn, seg_gt, lse, counts)
        ctx.mark_non_differentiable(counts)
        return loss, counts

    @staticmethod
    def backward(ctx, grad_loss, _grad_counts):
        fcn, seg, lse, counts = ctx.saved_tensors
        _, S, h, w = fcn.shape
        dfcn = torch.empty_like(fcn)
        call("semantic_loss_backward", fcn.device, fcn, S, h, w, seg, int(seg.dtype == torch.int64), lse, counts,
             _grad(grad_loss, fcn.device), dfcn)
        return dfcn, None


class SemanticLoss(torch.nn.Module):
    """The semantic head's loss of one training image (models/fcn.py:101 + models/resnet_upsnet.py:79,131):
    CrossEntropyLoss(ignore_index=255)(F.interpolate(fcn_score, scale_factor=4, mode='bilinear', align_corners=False),
    seg_gt), with the x4 up-sampling evaluated inside the loss (the logits are ops.upsample_bilinear's, bit for bit), so
    the [1,S,4h,4w] tensor, its log-softmax and its gradient are never built.  Backward keeps 4 bytes per output pixel.

    A label that is neither 255 nor a channel (torch asserts on it) gives no loss and no gradient; self.counts, int32 [2]
    on the device, is (pixels in the mean, such invalid pixels).  When every pixel is ignored the loss is NaN and the
    gradient zero, as torch's.  The same inputs give the same bytes."""

    def forward(self, fcn_score, seg_gt):
        """fcn_score [1,S,h,w] (float32; other float dtypes are cast); seg_gt [1,4h,4w] int64 or uint8.  -> loss, a
        0-dim device tensor."""
        E = _lib.UpsnetError
        require_cuda(fcn_score, seg_gt)
        if fcn_score.dim() != 4 or fcn_score.shape[0] != 1:
            raise E("semantic_loss: only batch size 1 (fcn_score [1,S,h,w])")
        _, S, h, w = fcn_score.shape
        if seg_gt.dim() != 3 or tuple(seg_gt.shape) != (1, 4 * h, 4 * w):
            raise E("semantic_loss: seg_gt must be [1,%d,%d] (four times fcn_score's size), not %s"
                    % (4 * h, 4 * w, tuple(seg_gt.shape)))
        if seg_gt.dtype not in (torch.int64, torch.uint8):
            raise E("semantic_loss: seg_gt must be int64 or uint8")
        loss, counts = SemanticLossFunction.apply(fcn_score, seg_gt.contiguous())
        self.counts = counts
        return loss


class FcnRoiLossFunction(torch.autograd.Function):
    """(loss, counts) = the fused FCN ROI loss (include/upsnet_b200.h, upsnet_fcn_roi_loss_forward); differentiable in
    fcn_score and score_bias.  Inputs are validated by FcnRoiLoss.forward."""

    @staticmethod
    def forward(ctx, fcn_score, score_bias, rois, seg_roi_gt, mask_size, spatial_scale):
        dev = fcn_score.device
        _, S, h, w = fcn_score.shape
        R = rois.shape[0]
        fcn, bias = f32c(fcn_score.detach()), f32c(score_bias.detach())
        (loss,) = _scalars(dev, 1)
        counts = torch.empty(2, dtype=torch.int32, device=dev)
        lse = torch.empty(R * mask_size * mask_size, dtype=torch.float32, device=dev)
        ws = torch.empty(query_bytes("fcn_roi_loss_workspace_bytes", S, R, mask_size, 0), dtype=torch.uint8, device=dev)
        is64 = int(seg_roi_gt.dtype == torch.int64)
        call("fcn_roi_loss_forward", dev, fcn, bias, S, h, w, rois, R, seg_roi_gt, is64, mask_size, 2, spatial_scale,
             loss, counts, lse, ws, ws.numel())
        ctx.save_for_backward(fcn, bias, rois, seg_roi_gt, lse)
        ctx.cfg = (mask_size, spatial_scale)
        ctx.mark_non_differentiable(counts)
        return loss, counts

    @staticmethod
    def backward(ctx, grad_loss, _grad_counts):
        fcn, bias, rois, seg, lse = ctx.saved_tensors
        M, scale = ctx.cfg
        dev = fcn.device
        _, S, h, w = fcn.shape
        R = rois.shape[0]
        dfcn, dbias = torch.empty_like(fcn), torch.empty_like(bias)
        ws = torch.empty(query_bytes("fcn_roi_loss_workspace_bytes", S, R, M, 1), dtype=torch.uint8, device=dev)
        call("fcn_roi_loss_backward", dev, fcn, bias, S, h, w, rois, R, seg, int(seg.dtype == torch.int64), M, 2, scale,
             lse, _grad(grad_loss, dev), dfcn, dbias, ws, ws.numel())
        return dfcn, dbias, None, None, None, None


class FcnRoiLoss(torch.nn.Module):
    """The semantic head's ROI loss of one training image (train.fcn_with_roi_loss; models/fcn.py:102-106 +
    models/resnet_upsnet.py:132-134): CrossEntropyLoss(ignore_index=255, reduce=False)(score(RoIAlign(M, M, 1/4)(feat,
    rois)), seg_roi_gt).mean(), with feat the 512-channel concat of the head.  The 1x1 score conv and ROIAlign commute,
    so the loss samples fcn_score (the score conv's output at quarter resolution) and adds the part of score_bias that
    ROIAlign's out-of-map zeros remove; feat, the [R,512,M,M] roi features and their gradients are never built.

    The mean runs over all R*M*M cells, ignored ones included, as the reference's.  A target that is neither 255 nor a
    class gives no loss and no gradient; self.counts, int32 [2] on the device, is (cells with a target, such invalid
    cells).  The loss is differentiable in fcn_score and score_bias; nothing synchronises with the host, so the call can
    be captured.  The same inputs give the same bytes."""

    def __init__(self, mask_size=28, spatial_scale=0.25):
        super().__init__()
        self.mask_size, self.spatial_scale = int(mask_size), float(spatial_scale)

    def forward(self, fcn_score, score_bias, rois, seg_roi_gt):
        """fcn_score [1,S,h,w] (float32; other float dtypes are cast); score_bias [S]; rois float32 [R,5] (batch index,
        x1, y1, x2, y2 in image coordinates, as gt_rois gives them), 1 <= R <= 1024; seg_roi_gt [R,M,M] int64 or uint8.
        -> loss, a 0-dim device tensor."""
        E = _lib.UpsnetError
        require_cuda(fcn_score, score_bias, rois, seg_roi_gt)
        M = self.mask_size
        if fcn_score.dim() != 4 or fcn_score.shape[0] != 1:
            raise E("fcn_roi_loss: only batch size 1 (fcn_score [1,S,h,w])")
        S = fcn_score.shape[1]
        if tuple(score_bias.shape) != (S,):
            raise E("fcn_roi_loss: score_bias must be [%d], not %s" % (S, tuple(score_bias.shape)))
        if rois.dim() != 2 or rois.shape[1] != 5 or rois.dtype != torch.float32:
            raise E("fcn_roi_loss: rois must be float32 [R,5], not %s %s" % (rois.dtype, tuple(rois.shape)))
        R = rois.shape[0]
        if tuple(seg_roi_gt.shape) != (R, M, M):
            raise E("fcn_roi_loss: seg_roi_gt must be [%d,%d,%d] (one row per roi), not %s"
                    % (R, M, M, tuple(seg_roi_gt.shape)))
        if seg_roi_gt.dtype not in (torch.int64, torch.uint8):
            raise E("fcn_roi_loss: seg_roi_gt must be int64 or uint8")
        loss, counts = FcnRoiLossFunction.apply(fcn_score, score_bias, rois.contiguous(), seg_roi_gt.contiguous(), M,
                                                self.spatial_scale)
        self.counts = counts
        return loss


def _carray(ctype, values):
    return (ctype * len(values))(*values)


class RPNLossFunction(torch.autograd.Function):
    """(cls_loss, bbox_loss) = the fused RPN loss (include/upsnet_b200.h, upsnet_rpn_loss_forward), differentiable in
    every level's score and box prediction.  `fields` holds the per-level label maps and their strides; inputs are
    validated by RPNLoss.forward."""

    @staticmethod
    def forward(ctx, fields, batch, *maps):
        L = len(maps) // 2
        scores, preds = [f32c(m.detach()) for m in maps[:L]], [f32c(m.detach()) for m in maps[L:]]
        dev = scores[0].device
        A = scores[0].shape[1]
        args = RPNLossFunction._args(scores, preds, fields)
        total = A * sum(s.shape[2] * s.shape[3] for s in scores)
        cls_loss, bbox_loss = _scalars(dev, 2)
        ws = torch.empty(query_bytes("rpn_loss_workspace_bytes", total), dtype=torch.uint8, device=dev)
        call("rpn_loss_forward", dev, L, A, *args, float(batch), cls_loss, bbox_loss, ws, ws.numel())
        ctx.save_for_backward(*scores, *preds)
        ctx.fields, ctx.batch = fields, batch
        return cls_loss, bbox_loss

    @staticmethod
    def _args(scores, preds, fields):
        """The per-level host arrays of the C call, from h / w through bbox_strides."""
        ptrs = lambda ts: _carray(C.c_void_p, [t.data_ptr() for t in ts])  # noqa: E731
        lab, tgt, iw, ow, lst, bst = fields
        return (_carray(C.c_int, [s.shape[2] for s in scores]), _carray(C.c_int, [s.shape[3] for s in scores]),
                ptrs(scores), ptrs(preds), ptrs(lab), _carray(C.c_longlong, lst), ptrs(tgt), ptrs(iw), ptrs(ow),
                _carray(C.c_longlong, bst))

    @staticmethod
    def backward(ctx, grad_cls, grad_bbox):
        t = ctx.saved_tensors
        L = len(t) // 2
        scores, preds = list(t[:L]), list(t[L:])
        dev = scores[0].device
        want_s = any(ctx.needs_input_grad[2:2 + L])
        want_p = any(ctx.needs_input_grad[2 + L:])
        ds = [torch.empty_like(s) for s in scores] if want_s else None
        dp = [torch.empty_like(p) for p in preds] if want_p else None
        if want_s or want_p:
            ptrs = lambda ts: _carray(C.c_void_p, [x.data_ptr() for x in ts]) if ts is not None else None  # noqa: E731
            call("rpn_loss_backward", dev, L, scores[0].shape[1], *RPNLossFunction._args(scores, preds, ctx.fields),
                 float(ctx.batch), _grad(grad_cls, dev), _grad(grad_bbox, dev), ptrs(ds), ptrs(dp))
        return (None, None) + tuple(ds if want_s else [None] * L) + tuple(dp if want_p else [None] * L)


class RPNLoss(torch.nn.Module):
    """RPNLoss.forward of models/rpn.py:60-92 (with_fpn) for one image, all FPN levels in one launch forward and one
    backward: BCE-with-logits of the scores against the labels (weight label != -1, sum / rpn_batch_size) and the
    smooth-L1 (sigma 3) of the box predictions with inside / outside weights (sum / batch, batch 1), each summed over the
    levels.  The label dict is RPNTargets' (or the reference loader's, on the device); its F x F field maps are read in
    place through their strides where the reference slices [:, :, :h, :w].  Built from the reference's `config`
    (train.rpn_batch_size * train.batch_size, as models/resnet_upsnet.py:79 does) or `rpn_batch_size`.  The same inputs
    give the same bytes."""

    STRIDES = (4, 8, 16, 32, 64)

    def __init__(self, config=None, *, rpn_batch_size=256):
        super().__init__()
        if config is not None:
            rpn_batch_size = config.train.rpn_batch_size * config.train.batch_size
        self.rpn_batch_size = int(rpn_batch_size)

    def forward(self, rpn_cls_score, rpn_bbox_pred, label):
        """rpn_cls_score / rpn_bbox_pred: the per-level lists [1,A,h,w] / [1,4A,h,w], strides 4, 8, ... in order;
        label: dict with 'rpn_labels_fpn{s}' [1,A,F,F] and 'rpn_bbox_{targets,inside_weights,outside_weights}_fpn{s}'
        [1,4A,F,F], F >= h, w.  -> (cls_loss, bbox_loss), 0-dim device tensors."""
        E = _lib.UpsnetError
        scores, preds = list(rpn_cls_score), list(rpn_bbox_pred)
        if not scores or len(scores) != len(preds) or len(scores) > len(self.STRIDES):
            raise E("rpn_loss: one score and one box map per level, at most %d levels" % len(self.STRIDES))
        require_cuda(*scores, *preds)
        A = scores[0].shape[1]
        lab, tgt, iw, ow, lst, bst = [], [], [], [], [], []
        for s, p, st in zip(scores, preds, self.STRIDES):
            if s.dim() != 4 or s.shape[0] != 1 or p.dim() != 4 or p.shape[0] != 1:
                raise E("rpn_loss: only batch size 1 (score [1,A,h,w], box prediction [1,4A,h,w])")
            h, w = s.shape[2:]
            if s.shape[1] != A or tuple(p.shape[1:]) != (4 * A, h, w):
                raise E("rpn_loss: stride %d: score %s and box prediction %s do not match" % (st, tuple(s.shape),
                                                                                            tuple(p.shape)))
            try:
                lv = [label[k % st] for k in ("rpn_labels_fpn%d", "rpn_bbox_targets_fpn%d",
                                               "rpn_bbox_inside_weights_fpn%d", "rpn_bbox_outside_weights_fpn%d")]
            except KeyError as e:
                raise E("rpn_loss: label has no %s" % e) from None
            require_cuda(*lv)
            for f, ch in zip(lv, (A, 4 * A, 4 * A, 4 * A)):
                if f.dim() != 4 or f.shape[0] != 1 or f.shape[1] != ch:
                    raise E("rpn_loss: stride %d: label field %s is not [1,%d,F,F]" % (st, tuple(f.shape), ch))
                if f.shape[2] < h or f.shape[3] < w:
                    raise E("rpn_loss: stride %d: label field %s is smaller than the %dx%d map" % (st, tuple(f.shape), h, w))
            l0 = lv[0] if lv[0].dtype == torch.int64 else lv[0].to(torch.int64)
            box = [f if f.dtype == torch.float32 else f.float() for f in lv[1:]]
            if l0.stride(3) != 1:
                l0 = l0.contiguous()
            if any(b.stride() != box[0].stride() or b.shape != box[0].shape or b.stride(3) != 1 for b in box):
                box = [b.contiguous() for b in box]
            lab.append(l0); tgt.append(box[0]); iw.append(box[1]); ow.append(box[2])
            lst += [l0.stride(1), l0.stride(2)]
            bst += [box[0].stride(1), box[0].stride(2)]
        return RPNLossFunction.apply((lab, tgt, iw, ow, lst, bst), self.rpn_batch_size, *scores, *preds)


class MaskRCNNLossFunction(torch.autograd.Function):
    """(cls_loss, bbox_loss, mask_loss, accuracy, counts) = the fused Mask R-CNN loss (include/upsnet_b200.h,
    upsnet_mask_rcnn_loss_forward), differentiable in cls_score, bbox_pred and mask_score.  Inputs are validated by
    MaskRCNNLoss.forward."""

    @staticmethod
    def forward(ctx, cls_score, bbox_pred, mask_score, cls_label, bbox_target, iw, ow, mask_target):
        cls, pred, msk = f32c(cls_score.detach()), f32c(bbox_pred.detach()), f32c(mask_score.detach())
        dev = cls.device
        R, K = cls.shape
        B, n = pred.shape[1], msk.numel()
        outs = _scalars(dev, 4)
        counts = torch.empty(4, dtype=torch.int32, device=dev)
        ws = torch.empty(query_bytes("mask_rcnn_loss_workspace_bytes", R, B, n), dtype=torch.uint8, device=dev)
        args = (cls, cls_label, R, K, pred, bbox_target, iw, ow, B, msk if n else None, mask_target if n else None, n)
        call("mask_rcnn_loss_forward", dev, *args, *outs, counts, ws, ws.numel())
        ctx.save_for_backward(cls, cls_label, pred, bbox_target, iw, ow, msk, mask_target, counts)
        ctx.mark_non_differentiable(outs[3], counts)
        return (*outs, counts)

    @staticmethod
    def backward(ctx, grad_cls, grad_bbox, grad_mask, _grad_acc, _grad_counts):
        cls, lab, pred, tgt, iw, ow, msk, mtgt, counts = ctx.saved_tensors
        dev = cls.device
        R, K = cls.shape
        B, n = pred.shape[1], msk.numel()
        need = ctx.needs_input_grad
        dcls = torch.empty_like(cls) if need[0] else None
        dpred = torch.empty_like(pred) if need[1] else None
        dmsk = torch.empty_like(msk) if need[2] else None
        if need[0] or need[1] or (need[2] and n):
            call("mask_rcnn_loss_backward", dev, cls, lab, R, K, pred, tgt, iw, ow, B, msk if n else None,
                 mtgt if n else None, n, counts, _grad(grad_cls, dev), _grad(grad_bbox, dev), _grad(grad_mask, dev),
                 dcls, dpred, dmsk if n else None)
        return (dcls, dpred, dmsk) + (None,) * 5


class MaskRCNNLoss(torch.nn.Module):
    """MaskRCNNLoss.forward of models/rcnn.py:159-197 for one image, one fused launch forward and one backward:
    cross-entropy with ignore_index -1 (mean over the other rows), smooth-L1 (sigma 1, sum / R), rcnn_accuracy exactly as
    written ((correct - ignored) / (R - ignored), the ignored rows subtracted from the correct ones too) and the mask loss
    sum(w (-x (t - b) + log(1 + exp(x - 2 x b)))) / (sum(w) + 1e-10), w = (t != -1), b = (x >= 0).  Takes the outputs of
    ProposalTargets.from_roidb unchanged.  self.counts, int32 [4] on the device: (rows in the mean, rows labelled -1, rows
    whose arg-max equals the label, mask elements with a target).  `batch_size` is accepted for the reference's
    signature and, as there, unused.  The same inputs give the same bytes."""

    def __init__(self, batch_size=None):
        super().__init__()
        self.counts = None

    def forward(self, cls_score, bbox_pred, mask_score, cls_label, bbox_target, bbox_inside_weight, bbox_outside_weight,
                mask_target):
        """cls_score [R,K]; bbox_pred and the three box tensors [R,B]; mask_score [n,K,M,M]; cls_label [R] (int64;
        -1 ignored); mask_target [n,K*M*M] (or any shape of as many elements; -1 ignored).  -> (cls_loss, bbox_loss,
        mask_loss, accuracy), 0-dim device tensors."""
        E = _lib.UpsnetError
        box = (bbox_target, bbox_inside_weight, bbox_outside_weight)
        require_cuda(cls_score, bbox_pred, mask_score, cls_label, mask_target, *box)
        if cls_score.dim() != 2 or cls_score.shape[0] == 0:
            raise E("mask_rcnn_loss: cls_score must be [R,K] with R >= 1")
        R = cls_score.shape[0]
        if cls_label.numel() != R:
            raise E("mask_rcnn_loss: cls_label must have one entry per cls_score row")
        if bbox_pred.dim() != 2 or bbox_pred.shape[0] != R or any(tuple(b.shape) != tuple(bbox_pred.shape) for b in box):
            raise E("mask_rcnn_loss: bbox_pred and the box targets / weights must all be [R,B]")
        if mask_score.dim() != 4 or mask_target.numel() != mask_score.numel() or (
                mask_target.dim() and mask_target.shape[0] != mask_score.shape[0]):
            raise E("mask_rcnn_loss: mask_target must have mask_score's rows and elements ([n,K*M*M] for [n,K,M,M])")
        loss = MaskRCNNLossFunction.apply(cls_score, bbox_pred, mask_score, cls_label.to(torch.int64).reshape(-1).contiguous(),
                                          *[f32c(b) for b in box], f32c(mask_target))
        self.counts = loss[4]
        return loss[:4]


# ------------------------------------------------------------------------------------------------
# panoptic training labels
# ------------------------------------------------------------------------------------------------
def _nearest(n, fx, n_out=None):
    """cv2.resize(INTER_NEAREST) source indices along an axis of length n: by a scale fx (output cvRound(n * fx)), or
    to a size n_out (cv2's scale is then n_out / n in double)."""
    from .operators import label_restore_index
    if n_out is None:
        n_out = int(np.rint(n * fx))
    else:
        fx = n_out / float(n)
    if n_out == n:                      # cv2.resize copies when the size does not change, whatever fx is
        return np.arange(n, dtype=np.int32)
    return label_restore_index(n_out, fx, n).astype(np.int32)


def _pad_table(t, n):
    out = np.full(n, -1, np.int32)
    out[:len(t)] = t
    return out


class PackedLabels:
    """One roidb entry's instance polygons on the device (PanopticLabels.pack_roidb): views of one int32 upload, plus
    the host-side boxes of seg_roi_gt and the vertex counts the limits are checked against."""

    def __init__(self, buf, parts, G, roi_boxes, max_poly_verts, max_obj_verts):
        self.buf, self.G, self.roi_boxes = buf, G, roi_boxes
        self.max_poly_verts, self.max_obj_verts = max_poly_verts, max_obj_verts
        for name, (off, n, _) in parts.items():
            setattr(self, name, buf[off:off + n])


class PanopticLabels:
    """The label maps of the semantic and panoptic heads of one training image on the device: the label block of the
    reference's loaders (dataset/cityscapes.py:166-189, dataset/coco.py:151-187) and collate / gt_list_to_blob
    (dataset/base_dataset.py:925-976), bit-exact to them with Pillow 12.2 and cv2 4.13.

    seg_gt / seg_gt_4x / seg_roi_gt are gathers from the uint8 label map through cv2 INTER_NEAREST index tables built
    on the host (the flip folded into the columns); mask_gt evaluates Pillow's polygon fill only at the canvas pixels
    the two nearest resizes sample (csrc/labels.cu).  Built from the reference's `config` (network.mask_size,
    network.rpn_feat_stride[-2], train.fcn_with_roi_loss) or from the same values as keywords.  `dataset` selects the
    loader: "cityscapes" draws every roidb row and sizes the canvas int(blob / scale); "coco" draws the non-crowd
    rows, sizes it np.round(blob / scale), and keeps only non-crowd boxes for seg_roi_gt."""

    def __init__(self, config=None, *, dataset="cityscapes", mask_size=28, with_roi=None, stride=32):
        if dataset not in ("cityscapes", "coco"):
            raise _lib.UpsnetError("panoptic_labels: dataset must be 'cityscapes' or 'coco'")
        if config is not None:
            mask_size, stride = config.network.mask_size, config.network.rpn_feat_stride[-2]
            if with_roi is None:
                with_roi = config.train.fcn_with_roi_loss
        self.dataset, self.M, self.stride = dataset, int(mask_size), int(stride)
        self.with_roi = bool(with_roi)

    def _rows(self, entry):
        cls = np.asarray(entry["gt_classes"])
        crowd = np.asarray(entry["is_crowd"])
        if self.dataset == "cityscapes":
            return np.arange(len(cls)), np.where(cls > 0)[0]
        return np.where(crowd == 0)[0], np.where((cls > 0) & (crowd == 0))[0]

    def pack_roidb(self, entry, im_scale, device):
        """One upload of the polygons drawn into mask_gt (ProposalTargets' layout, vertices truncated toward zero to
        int32 as Pillow does), and the seg_roi_gt boxes np.around(boxes * im_scale).astype(int32) with the reference's
        +1 for a degenerate side (host-side)."""
        draw, roi_rows = self._rows(entry)
        obj_off, poly_off, polys = pack_polygons(entry["segms"], draw, "panoptic_labels")
        verts = [np.trunc(p).astype(np.int32) for ps in polys for p in ps]
        yr = np.zeros((len(polys), 2), np.int32)
        for g, ps in enumerate(polys):
            ys = np.concatenate([np.trunc(p[1::2]) for p in ps])
            yr[g] = (ys.min(), ys.max())
        sizes = np.diff(poly_off)
        per_obj = [int(sizes[obj_off[g]:obj_off[g + 1]].sum()) for g in range(len(polys))]
        boxes = None
        if self.with_roi:
            boxes = np.around(np.asarray(entry["boxes"])[roi_rows] * float(im_scale)).astype(np.int32).reshape(-1, 4)
            for b in boxes:
                if b[3] == b[1]:
                    b[3] += 1
                if b[2] == b[0]:
                    b[2] += 1
        arrays = [("obj_poly", obj_off, np.int32), ("poly_vert", poly_off, np.int32),
                  ("verts", np.concatenate(verts) if verts else np.zeros(2, np.int32), np.int32),
                  ("obj_yrange", yr.ravel(), np.int32)]
        buf, parts = _upload_parts(arrays, device)
        return PackedLabels(buf, parts, len(polys), boxes, int(sizes.max()) if sizes.size else 0,
                            max(per_obj) if per_obj else 0)

    def tables(self, label_shape, packed, im_shape, im_scale, flipped):
        """The int32 index tables of one call (host): {name: array} in label-map coordinates, -1 = padding, and the
        output shapes.  Raises where the reference fails: a canvas whose resize is not the blob's size, an empty
        seg_roi_gt crop."""
        s, st = float(im_scale), self.stride
        h0, w0 = label_shape
        rows, cols = _nearest(h0, s), _nearest(w0, s)
        if flipped:
            cols = (w0 - 1 - cols).astype(np.int32)
        h, w = len(rows), len(cols)
        Hp, Wp = int(np.ceil(h / float(st)) * st), int(np.ceil(w / float(st)) * st)
        qr, qc = _nearest(h, 0.25), _nearest(w, 0.25)
        t = {"seg_rows": _pad_table(rows, Hp), "seg_cols": _pad_table(cols, Wp),
             "q_rows": _pad_table(rows[qr], int(Hp * 0.25)), "q_cols": _pad_table(cols[qc], int(Wp * 0.25))}
        Hb, Wb = (int(v) for v in im_shape)
        if self.dataset == "cityscapes":
            Hc, Wc = int(Hb / s), int(Wb / s)
        else:
            Hc, Wc = int(np.round(Hb / s)), int(np.round(Wb / s))
        cr, cc = _nearest(Hc, s), _nearest(Wc, s)
        if (len(cr), len(cc)) != (Hb, Wb):
            raise _lib.UpsnetError("panoptic_labels: the %dx%d canvas resized by %r is %dx%d, not the blob's %dx%d"
                                   % (Hc, Wc, s, len(cr), len(cc), Hb, Wb))
        Hbp, Wbp = int(np.ceil(Hb / float(st)) * st), int(np.ceil(Wb / float(st)) * st)
        t["m_rows"] = _pad_table(cr[_nearest(Hb, 0.25)], int(Hbp * 0.25))
        t["m_cols"] = _pad_table(cc[_nearest(Wb, 0.25)], int(Wbp * 0.25))
        n = 0
        if self.with_roi:
            b = packed.roi_boxes
            n = len(b)
            rr, rc = np.zeros((n, self.M), np.int32), np.zeros((n, self.M), np.int32)
            ar, ac = np.arange(h), np.arange(w)
            for i in range(n):
                ys, xs = ar[b[i][1]:b[i][3]], ac[b[i][0]:b[i][2]]
                if ys.size == 0 or xs.size == 0:
                    raise _lib.UpsnetError("panoptic_labels: seg_roi_gt box %d crops nothing (cv2.resize raises)" % i)
                rr[i] = rows[ys[_nearest(ys.size, None, self.M)]]
                rc[i] = cols[xs[_nearest(xs.size, None, self.M)]]
            t["roi_rows"], t["roi_cols"] = rr.ravel(), rc.ravel()
        return t, n

    def prepare(self, label_shape, packed, im_shape, im_scale, flipped, device):
        """tables() uploaded in one copy: the device half of a call, so that `launch` issues kernels only (and can be
        captured in a CUDA graph)."""
        t, n = self.tables(label_shape, packed, im_shape, im_scale, flipped)
        buf, parts = _upload_parts([(k, v, np.int32) for k, v in t.items()], device)
        tab = {k: buf[off:off + m] for k, (off, m, _) in parts.items()}
        tab["n_roi"], tab["label_shape"] = n, tuple(label_shape)
        return tab

    def launch(self, label_map, packed, tab, mask_dtype=torch.uint8):
        """The kernels of one call on prepared tables; -> the dict of __call__."""
        require_cuda(label_map)
        if label_map.dim() != 2 or label_map.dtype != torch.uint8:
            raise _lib.UpsnetError("panoptic_labels: label_map must be uint8 [h0,w0]")
        if tuple(label_map.shape) != tab["label_shape"]:
            raise _lib.UpsnetError("panoptic_labels: the tables were prepared for another label map size")
        if mask_dtype not in (torch.uint8, torch.int64):
            raise _lib.UpsnetError("panoptic_labels: mask_dtype must be uint8 or int64")
        lab = label_map.contiguous()
        dev = lab.device
        n = tab["n_roi"]
        Hs, Ws, Hq, Wq = (tab[k].numel() for k in ("seg_rows", "seg_cols", "q_rows", "q_cols"))
        Hm, Wm, G = tab["m_rows"].numel(), tab["m_cols"].numel(), packed.G
        out = {"seg_gt": torch.empty((1, Hs, Ws), dtype=torch.int64, device=dev),
               "seg_gt_4x": torch.empty((1, Hq, Wq), dtype=torch.int64, device=dev),
               "mask_gt": torch.empty((G, Hm, Wm), dtype=mask_dtype, device=dev)}
        if self.with_roi:
            out["seg_roi_gt"] = torch.empty((n, self.M, self.M), dtype=torch.int64, device=dev)
        pk = packed
        call("training_labels", dev, lab, lab.shape[0], lab.shape[1], tab["seg_rows"], Hs, tab["seg_cols"], Ws,
             out["seg_gt"], tab["q_rows"], Hq, tab["q_cols"], Wq, out["seg_gt_4x"],
             tab["m_rows"], Hm, tab["m_cols"], Wm, pk.obj_poly, pk.poly_vert, pk.verts,
             pk.obj_yrange, G, pk.max_poly_verts, pk.max_obj_verts,
             out["mask_gt"] if G else None, int(mask_dtype == torch.int64),
             tab["roi_rows"] if n else None, tab["roi_cols"] if n else None, n, self.M,
             out["seg_roi_gt"] if n else None)
        return out

    def __call__(self, label_map, packed, im_shape, im_scale, flipped, mask_dtype=torch.uint8):
        """label_map: CUDA uint8 [h0,w0] (the decoded label PNG, not flipped); packed: pack_roidb's; im_shape: the
        resized image's (h, w) (get_image_blob); im_scale: im_scales[0], a Python float; flipped: the entry's flag.
        -> dict of device tensors: seg_gt int64 [1,Hp,Wp], seg_gt_4x int64 [1,Hp/4,Wp/4], mask_gt mask_dtype (uint8
        or int64; 0 / 1, 255 in the padding) [G,Hb_p/4,Wb_p/4], and seg_roi_gt int64 [n,M,M] when with_roi."""
        require_cuda(label_map)
        tab = self.prepare(tuple(label_map.shape), packed, im_shape, im_scale, flipped, label_map.device)
        return self.launch(label_map, packed, tab, mask_dtype)

    def from_roidb(self, entry, label_map, im_shape, im_scale, device):
        """Drop-in for the loader's label block and collate: {'seg_gt', 'seg_gt_4x', 'mask_gt' (int64), and
        'seg_roi_gt' when with_roi} with the reference's shapes and dtypes.  label_map: the decoded label PNG (uint8
        numpy array or tensor), not flipped; the flip is entry['flipped']."""
        lab = label_map if torch.is_tensor(label_map) else torch.from_numpy(np.ascontiguousarray(label_map, np.uint8))
        packed = self.pack_roidb(entry, im_scale, device)
        return self(lab.to(device), packed, im_shape, im_scale, bool(entry["flipped"]), mask_dtype=torch.int64)


# ------------------------------------------------------------------------------------------------
# one training sample: the loader's __getitem__ (phase train) + collate
# ------------------------------------------------------------------------------------------------
class TrainingSample:
    """The (data, label) pair the reference's DataLoader yields for one roidb entry (dataset/cityscapes.py:117-193,
    dataset/coco.py:124-191 with phase 'train', and collate, dataset/base_dataset.py:952-988), built on the device:

      data  = {'data': float32 [1,3,Hp,Wp] (prep_image, flipped as the entry says), 'im_info': numpy float32 [1,3]}
      label = {'roidb': the entry's minimal roidb (add_rpn_blobs' valid_keys), the RPN fields of RPNTargets,
               'seg_gt', 'seg_gt_4x', 'mask_gt' (int64), 'seg_roi_gt' with train.fcn_with_roi_loss (PanopticLabels),
               'gt_classes': every row (cityscapes) or the non-crowd rows (coco), in the entry's dtype}

    The scale is drawn as get_image_blob draws it, np.random.randint(0, high=len(scales), size=1), and capped by
    prep_im_for_blob's max_size rule in float64, so under the same np.random state the reference and this class train
    at the same scale; the RPN subsampling seed is drawn after it (RPNTargets).  Built from the reference's `config`
    (train.scales, train.max_size, network.pixel_means, network.rpn_feat_stride[-2], and what RPNTargets and
    PanopticLabels read) or from the same values as keywords (the rest go to RPNTargets); `dataset` selects the loader,
    "cityscapes" or "coco".

    Not built here: data_4x (collate makes it, no module of the model reads it); the image and PNG decoding (host);
    RLE segmentations (PanopticLabels rejects them); the flipped entries themselves (extend_with_flipped_entries: a
    flipped entry carries flipped boxes and segms and flipped=True); any stream or prefetch machinery."""

    ROIDB_KEYS = ("boxes", "segms", "seg_areas", "gt_classes", "gt_overlaps", "is_crowd", "box_to_gt_ind_map")

    def __init__(self, config=None, *, dataset="cityscapes", scales=(800,), max_size=1333,
                 pixel_means=(102.9801, 115.9465, 122.7717), stride=32, mask_size=28, with_roi=None, **rpn):
        if config is not None:
            if not config.network.use_caffe_model:
                raise _lib.UpsnetError("training_sample: only network.use_caffe_model (mean subtraction) is built")
            scales, max_size = config.train.scales, config.train.max_size
            pixel_means, stride = config.network.pixel_means, config.network.rpn_feat_stride[-2]
            self.rpn = RPNTargets(config)
            self.labels = PanopticLabels(config, dataset=dataset, with_roi=with_roi)
        else:
            self.rpn = RPNTargets(max_size=max_size, **rpn)
            self.labels = PanopticLabels(dataset=dataset, mask_size=mask_size, with_roi=with_roi, stride=stride)
        if len(scales) == 0:
            raise _lib.UpsnetError("training_sample: no train.scales")
        self.scales, self.max_size = list(scales), max_size
        self.pixel_means = [float(v) for v in pixel_means]
        self.stride, self.dataset = int(stride), dataset

    def im_scale(self, target_size, h, w):
        """prep_im_for_blob's scale of an h x w image for one target size (base_dataset.py:158-168)."""
        return prep_scale(target_size, self.max_size, h, w)

    def draw_scale(self, h, w):
        """get_image_blob's draw (base_dataset.py:119-121) -> (scale index, im_scale)."""
        ind = int(np.random.randint(0, high=len(self.scales), size=1)[0])
        return ind, self.im_scale(self.scales[ind], h, w)

    def sample(self, entry, image_bgr_u8, label_map_u8, device, seed=None):
        """entry: a roidb entry; image_bgr_u8: the decoded image uint8 [h,w,3] and label_map_u8: the decoded label PNG
        uint8 [h,w], both as read from disk (not flipped), numpy arrays or tensors; seed: RPNTargets' subsampling seed
        (None draws it from np.random after the scale).  -> (data, label) as in the class docstring.  Bad input raises
        UpsnetError before any kernel is launched."""
        h, w = int(entry["height"]), int(entry["width"])
        im, lab = (x if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(x))
                   for x in (image_bgr_u8, label_map_u8))
        if im.dtype != torch.uint8 or tuple(im.shape) != (h, w, 3):
            raise _lib.UpsnetError("training_sample: the image is %s %s, the entry's is uint8 (%d, %d, 3)"
                                   % (im.dtype, tuple(im.shape), h, w))
        if lab.dtype != torch.uint8 or tuple(lab.shape) != (h, w):
            raise _lib.UpsnetError("training_sample: the label map is %s %s, the entry's is uint8 (%d, %d)"
                                   % (lab.dtype, tuple(lab.shape), h, w))
        cls, crowd = np.asarray(entry["gt_classes"]), np.asarray(entry["is_crowd"])
        if not ((cls > 0) & (crowd == 0)).any():
            raise _lib.UpsnetError("training_sample: no ground-truth boxes (add_rpn_blobs fails on such an entry)")
        _, s = self.draw_scale(h, w)
        ho, wo = int(np.rint(h * s)), int(np.rint(w * s))
        flipped = bool(entry["flipped"])
        # the host half of the label maps first: a polygon or canvas they reject raises before any launch
        packed = self.labels.pack_roidb(entry, s, device)
        tab = self.labels.prepare((h, w), packed, (ho, wo), s, flipped, device)
        blob, _ = prep_image(im.to(device, non_blocking=True), self.pixel_means, s, self.stride, flip=flipped)
        data = {"data": blob, "im_info": np.array([[np.round(h * s), np.round(w * s), s]], np.float32)}
        label = {"roidb": {k: entry[k] for k in self.ROIDB_KEYS if k in entry}}
        label.update(self.rpn.from_roidb(entry, s, device, seed))
        label.update(self.labels.launch(lab.to(device, non_blocking=True), packed, tab, mask_dtype=torch.int64))
        rows = np.arange(len(cls)) if self.dataset == "cityscapes" else np.flatnonzero(crowd == 0)
        label["gt_classes"] = torch.from_numpy(np.ascontiguousarray(cls[rows])).to(device)
        return data, label
