"""The training step of models/resnet_upsnet.py:88-195 in plain torch, differentiable -- TEST INFRASTRUCTURE ONLY,
independent of the product.

The graph is oracle/literal_model.py's LiteralUPSNet, the reference's graph restated literally; this module adds what
is about training: the trainable parameters and their gradients, conv1 / res2 frozen (backbone_freeze_at = 2), the
losses, and the planted faults.  The losses are the existing loss oracles (train_loss_oracle, panoptic_loss_oracle),
with the semantic head's cross-entropy taken on the x4 up-sampled score.  The discrete decisions of a step (proposals,
sampled targets, gt rois, keep_inds) are taken from the product's `_intermediates`, so the oracle replays the same
step.  Parameters are leaf tensors in any float dtype, on the CPU or the GPU.

The COCO configurations build the same oracle with with_gap (FPN's global context branch, models/fpn.py:84-86) and
fcn_with_roi_loss (the semantic head's ROI loss, models/fcn.py:102-106, models/resnet_upsnet.py:132-134, restated
literally: RoIAlign of the 512-channel concat, the score conv, the cross-entropy with ignore_index 255 averaged over
every cell, on the product's 'fcn_rois': every ground-truth box, before the keep draw).

`fault` plants one of FAULTS or COCO_FAULTS, for the tests that show the gradient criterion rejects it: 'gap_detached'
takes no gradient through fpn_gap, 'rois_after_keep' takes the ROI loss on the kept boxes and their seg_roi_gt rows.
"""
import numpy as np
import torch
import torch.nn.functional as F

import fcn_roi_loss_oracle as FO
import panoptic_loss_oracle as PO
import train_loss_oracle as TO
from oracle.literal_model import LiteralUPSNet

FAULTS = ("bn_scale_dw", "p6_grad", "fcn_level_detached", "pan_mask_grad", "res2_trainable")
COCO_FAULTS = ("gap_detached", "rois_after_keep")
STRIDES = (4, 8, 16, 32, 64)


def trainable_names(model):
    """The names of the parameters the reference trains: get_params_lr()'s, by name."""
    ids = {id(p) for g in model.get_params_lr() for p in g["params"]}
    return [n for n, p in model.named_parameters() if id(p) in ids]


def gap_vector(res5, weight, bias, detached=False):
    """models/fpn.py:85: fpn_gap(adaptive_avg_pool2d(res5, 1)) as [1, C, 1, 1]."""
    if detached:
        res5, weight, bias = res5.detach(), weight.detach(), bias.detach()
    return F.linear(F.adaptive_avg_pool2d(res5, (1, 1)).flatten(1), weight, bias).view(1, -1, 1, 1)


def roi_loss(feat, weight, bias, rois, seg, keep=None):
    """The reference's fcn_roi_loss from the 512-channel concat feat [1,512,h,w]; with keep, the faulty variant that
    takes only the kept boxes (and their rows)."""
    if keep is not None:
        keep = torch.as_tensor(keep, device=rois.device).long()
        rois, seg = rois[keep], seg[keep]
    f = feat[0]
    By, Bx, _ = FO.roi_align_weights(rois, f.shape[1], f.shape[2], seg.shape[1])
    rf = torch.einsum("rmy,cyx,rnx->rcmn", By.to(f.dtype), f, Bx.to(f.dtype))
    return FO.ce_mean(F.conv2d(rf, weight, bias), seg.long())


class TrainOracle(LiteralUPSNet):
    def __init__(self, state_dict, trainable, depth=(2, 2, 2, 2), rpn_batch_size=256, fcn_with_roi_loss=False,
                 dtype=torch.float64, fault=None, **kw):
        assert fault is None or fault in FAULTS + COCO_FAULTS
        self.fault = fault
        train = set(trainable)
        if fault == "res2_trainable":
            train |= {k for k in state_dict if k.startswith("resnet_backbone.res2.") and ".bn" not in k and
                      "downsample.1" not in k and not k.endswith(("running_mean", "running_var", "num_batches_tracked"))}
        super().__init__(state_dict, depth=depth, dtype=dtype, trainable=train, **kw)
        self.trainable = sorted(train)
        self.rpn_batch_size, self.fcn_with_roi_loss = rpn_batch_size, fcn_with_roi_loss

    def grads(self):
        return {k: (None if self.p[k].grad is None else self.p[k].grad.detach()) for k in self.trainable}

    # ------------------------------------------------------------------ the frozen stem and the planted faults
    def stem_res2(self, x):
        if self.fault == "res2_trainable":
            return super().stem_res2(x)
        with torch.no_grad():
            return super().stem_res2(x)

    def bn(self, x, name):
        y = super().bn(x, name)
        if self.fault == "bn_scale_dw":     # the value is right, the gradient skips the BN scale
            y = x + (y - x).detach()
        return y

    def gap(self, res5):
        return gap_vector(res5, self.p["fpn.fpn_gap.weight"], self.p["fpn.fpn_gap.bias"], self.fault == "gap_detached")

    def fpn(self, r2, r3, r4, r5):
        p = super().fpn(r2, r3, r4, r5)
        if self.fault == "p6_grad":
            p = p[:4] + (F.max_pool2d(p[3].detach(), 1, 2),)
        return p

    def fcn_level(self, x, level):
        x = super().fcn_level(x, level)
        return x.detach() if self.fault == "fcn_level_detached" and level == 2 else x

    # ------------------------------------------------------------------ the step
    def forward(self, image, label, inter):
        """image [1,3,H,W]; label: the loader's dict (rpn fields, seg_gt, seg_gt_4x, mask_gt, and seg_roi_gt with the
        ROI loss); inter: the product's _intermediates.  -> dict of the nine outputs, plus fcn_roi_loss with the ROI
        loss, as 0-dim tensors (accuracies as floats)."""
        dev, dt = self.device, self.dtype
        r2, r3, r4, r5 = self.backbone(image.to(dev, dt))
        fpn = self.fpn(r2, r3, r4, r5)
        rpn = [self.rpn(f) for f in fpn]
        rpn_cls = rpn_box = 0
        for (score, pred, _), s in zip(rpn, STRIDES):
            h, w = score.shape[2:]
            sl = lambda k: label[k % s].to(dev)[:, :, :h, :w]             # noqa: E731
            lab = sl("rpn_labels_fpn%d")
            rpn_cls = rpn_cls + F.binary_cross_entropy_with_logits(score, lab.to(dt), (lab != -1).to(dt),
                                                                   reduction="sum") / self.rpn_batch_size
            rpn_box = rpn_box + TO._smooth_l1(pred, sl("rpn_bbox_targets_fpn%d").to(dt),
                                              sl("rpn_bbox_inside_weights_fpn%d").to(dt),
                                              sl("rpn_bbox_outside_weights_fpn%d").to(dt), 3.0).sum()
        fcn = self.fcn_head(*fpn[:4])
        fcn_loss = TO.semantic_from_logits(fcn["fcn_output"], label["seg_gt"].to(dev))[0]

        t = inter["proposal_targets"]
        feats = list(fpn[:4])
        rcnn = self.rcnn(feats, t["rois"])
        cls_score, bbox_pred = rcnn["cls_score"], rcnn["bbox_pred"]
        lab = t["labels"].to(dev).long()
        cls_loss = F.cross_entropy(cls_score, lab, ignore_index=-1)
        box = TO._smooth_l1(bbox_pred, *(t[k].to(dev, dt) for k in ("bbox_targets", "bbox_inside_weights",
                                                                      "bbox_outside_weights")), 1.0)
        bbox_loss = box.sum() / box.shape[0]
        R = cls_score.shape[0]
        ignore = int((lab == -1).sum())
        rcnn_acc = (int((cls_score.detach().argmax(1) == lab).sum()) - ignore) / float(R - ignore)
        if t["mask_rois"].shape[0]:
            m = self.mask_branch(feats, t["mask_rois"])
            tgt = t["mask_int32"].to(dev, dt).view(m.shape)
            wgt = (tgt != -1).to(dt)
            b = (m >= 0).to(dt)
            mask_loss = ((-m * (tgt - b) + torch.log1p(torch.exp(m - 2 * m * b))) * wgt).sum() / (wgt.sum() + 1e-10)
        else:
            mask_loss = cls_loss.new_zeros(())

        gt_rois, cls_idx, keep = inter["gt_rois"], inter["cls_idx"], inter["keep_inds"]
        pm = self.mask_branch(feats, gt_rois)
        if self.fault == "pan_mask_grad":
            pm = pm.detach()
        logits = PO.panoptic_logits(fcn["fcn_score"].cpu().to(dt), pm.cpu().to(dt), gt_rois.detach().cpu().numpy(),
                                    cls_idx.cpu().numpy(), self.num_classes, keep is not None)
        gt = PO.panoptic_gt(label["seg_gt_4x"].cpu().numpy(), label["mask_gt"].cpu().numpy(),
                            None if keep is None else np.asarray(keep), self.num_seg_classes, self.num_classes)
        panoptic_loss, correct, ignored = PO.loss_and_accuracy(logits, gt)
        out = {"rpn_cls_loss": rpn_cls, "rpn_bbox_loss": rpn_box, "cls_loss": cls_loss, "bbox_loss": bbox_loss,
               "mask_loss": mask_loss, "fcn_loss": fcn_loss, "panoptic_loss": panoptic_loss.to(dev),
               "rcnn_accuracy": rcnn_acc, "panoptic_accuracy": correct / float(gt.size - ignored)}
        if self.fcn_with_roi_loss:
            rois, seg = inter["fcn_rois"].to(dev), label["seg_roi_gt"].to(dev)
            out["fcn_roi_loss"] = roi_loss(fcn["fcn_feat"], self.p["fcn_head.score.weight"], self.p["fcn_head.score.bias"],
                                           rois, seg, keep if self.fault == "rois_after_keep" else None)
        return out

    def step(self, image, label, inter):
        """forward + backward of the sum of the losses -> (outputs as floats, grads)."""
        out = self.forward(image, label, inter)
        total = sum(out[k] for k in COCO_LOSSES if k in out)
        total.backward()
        return {k: float(v.detach()) if torch.is_tensor(v) else float(v) for k, v in out.items()}, self.grads()


# per-tensor relative L2 error of a gradient, and relative error of a loss, allowed for the device step against the
# float64 oracle: about 4x the worst ratio measured on an H100 80GB HBM3 at 700 W (tests/test_gpu_train_forward.py).
# The offset convs of the deformable layers get their own bound: their gradient is the derivative of the bilinear
# sample in its position, which jumps where a sample crosses a pixel edge, so a rounding-level change of an offset
# moves a few samples' contributions between neighbouring pixels.
# Measured worst ratios: bf16x3 2.3e-3 (5.0e-3 in an offset conv), losses 5.1e-4; bf16 4.5e-2 (9.0e-2), losses 3.1e-3.
GRAD_TOL = {"bf16x3": 1e-2, "bf16": 0.2}
OFFSET_GRAD_TOL = {"bf16x3": 2e-2, "bf16": 0.35}
LOSS_TOL = {"bf16x3": 2e-3, "bf16": 1.5e-2}


def grad_tol(name, prec):
    return (OFFSET_GRAD_TOL if "offset" in name else GRAD_TOL)[prec]

LOSSES = ("rpn_cls_loss", "rpn_bbox_loss", "cls_loss", "bbox_loss", "mask_loss", "fcn_loss", "panoptic_loss")
COCO_LOSSES = LOSSES + ("fcn_roi_loss",)
OUTPUTS = LOSSES + ("rcnn_accuracy", "panoptic_accuracy")


def grad_errors(got, want):
    """{name: relative L2 error of got[name] against want[name]}; a gradient present on one side only is error inf
    (1.0 when both are zero)."""
    err = {}
    for k, w in want.items():
        g = got.get(k)
        if (g is None) != (w is None):
            err[k] = float("inf")
            continue
        if g is None:
            err[k] = 0.0
            continue
        g, w = g.double().cpu(), w.double().cpu()
        n = float(w.norm())
        err[k] = float((g - w).norm()) / n if n > 0 else (0.0 if float(g.norm()) == 0 else 1.0)
    extra = set(got) - set(want)
    for k in extra:
        if got[k] is not None:
            err[k] = float("inf")
    return err


# ------------------------------------------------------------------------------------------------
# seeded synthetic step
# ------------------------------------------------------------------------------------------------
def synthetic_entry(seed, h, w, G, num_classes=9):
    """A Cityscapes-like roidb entry of G star-polygon instances on an h x w image (scale 1), and its uint8 label map."""
    import label_oracle as LO
    rng = np.random.default_rng(seed)
    segms, boxes = [], []
    for _ in range(G):
        r = rng.uniform(min(h, w) / 12.0, min(h, w) / 4.0)
        cx, cy = rng.uniform(r, w - r), rng.uniform(r, h - r)
        ps = [LO.star(rng, cx, cy, r, int(rng.integers(5, 16)))]
        segms.append(ps)
        a = np.asarray(ps[0])
        boxes.append([a[0::2].min(), a[1::2].min(), a[0::2].max(), a[1::2].max()])
    boxes = np.asarray(boxes, np.float32)
    boxes[:, 0::2] = np.clip(boxes[:, 0::2], 0, w - 1)
    boxes[:, 1::2] = np.clip(boxes[:, 1::2], 0, h - 1)
    cls = rng.integers(1, num_classes, G).astype(np.int32)
    ov = np.zeros((G, num_classes), np.float32)
    ov[np.arange(G), cls] = 1
    entry = dict(boxes=boxes, gt_classes=cls, is_crowd=np.zeros(G, np.int32), segms=segms, flipped=False, height=h,
                 width=w, gt_overlaps=ov, box_to_gt_ind_map=np.arange(G, dtype=np.int32))
    return entry, LO.label_png(h, w, seed)


def image(seed, h, w):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(1, 3, h, w, generator=g) * 50


def fixture_values(seed, shape, scale=1.0, offset=0.0):
    """Deterministic float32 values, uniform in offset + scale * [-1/2, 1/2), defined by this code alone (splitmix64
    keys of upsnet_b200.training.draw_keys, top 24 bits): the FPN / RPN inputs and parameters of
    tests/golden/make_reference_group_norm.py, made again by the test instead of being stored in the fixture."""
    from upsnet_b200.training import draw_keys
    n = int(np.prod(shape))
    u = (draw_keys(seed, n) >> np.uint64(40)).astype(np.float64) / 2.0 ** 24
    return torch.from_numpy(((u - 0.5) * scale + offset).astype(np.float32).reshape(shape))


def fixture_fpn_params(shapes):
    """{name: tensor} for the (name, shape) list of the reference FPN / RPN parameters, in order: GroupNorm weights
    around 1, other biases and GN biases around 0 (scale 0.4), weights at scale 0.1."""
    out = {}
    for i, (name, shape) in enumerate(shapes):
        gn_w = name.endswith(".1.weight")
        out[name] = fixture_values(1000 + i, shape, 0.4 if len(shape) == 1 else 0.1, 1.0 if gn_w else 0.0)
    return out
