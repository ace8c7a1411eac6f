"""Differentiable restatement of the training forward of models/resnet_upsnet.py:88-195 in plain torch -- TEST
INFRASTRUCTURE ONLY, independent of the product as oracle/literal_model.py is.

The graph is written the way the reference writes it: un-folded frozen BatchNorm, conv1 / res2 detached
(backbone_freeze_at = 2), nearest-neighbour FPN up-sampling materialised, the semantic head as concat -> score -> x4
up-sampling inside the cross-entropy, ConvTranspose2d for the mask deconv, torchvision's deform_conv2d and roi_align for
the custom operators, and the existing loss oracles (train_loss_oracle, panoptic_loss_oracle).  The discrete decisions of
a step (proposals, sampled targets, gt rois, keep_inds) are taken from the product's `_intermediates`, so the oracle
replays the same step.  Parameters are leaf tensors in any float dtype, on the CPU or the GPU.

`fault` plants one of FAULTS, for the tests that show the gradient criterion rejects it.
"""
import numpy as np
import torch
import torch.nn.functional as F
import torchvision

import panoptic_loss_oracle as PO
import train_loss_oracle as TO

FAULTS = ("bn_scale_dw", "p6_grad", "fcn_level_detached", "pan_mask_grad", "res2_trainable")
STRIDES = (4, 8, 16, 32, 64)


def trainable_names(model):
    """The names of the parameters the reference trains: get_params_lr()'s, by name."""
    ids = {id(p) for g in model.get_params_lr() for p in g["params"]}
    return [n for n, p in model.named_parameters() if id(p) in ids]


class TrainOracle:
    def __init__(self, state_dict, trainable, depth=(2, 2, 2, 2), num_classes=9, num_seg_classes=19, dconv_from=100,
                 fcn_layers=2, rpn_batch_size=256, dtype=torch.float64, device="cpu", fault=None):
        assert fault is None or fault in FAULTS
        self.fault = fault
        train = set(trainable)
        if fault == "res2_trainable":
            train |= {k for k in state_dict if k.startswith("resnet_backbone.res2.") and ".bn" not in k and
                      "downsample.1" not in k and not k.endswith(("running_mean", "running_var", "num_batches_tracked"))}
        self.p = {}
        for k, v in state_dict.items():
            if k.endswith("num_batches_tracked"):
                continue
            t = v.detach().to(device=device, dtype=dtype).clone()
            self.p[k] = t.requires_grad_(k in train)
        self.trainable = sorted(train)
        self.depth, self.num_classes, self.num_seg_classes = depth, num_classes, num_seg_classes
        self.dconv_from, self.fcn_layers, self.rpn_batch_size = dconv_from, fcn_layers, rpn_batch_size
        self.dtype, self.device = dtype, device

    def grads(self):
        return {k: (None if self.p[k].grad is None else self.p[k].grad.detach()) for k in self.trainable}

    # ------------------------------------------------------------------ primitives
    def conv(self, x, name, stride=1, padding=0, dilation=1):
        return F.conv2d(x, self.p[name + ".weight"], self.p.get(name + ".bias"), stride, padding, dilation)

    def bn(self, x, name):          # frozen BatchNorm, eval mode, NOT folded
        s = self.p
        y = F.batch_norm(x, s[name + ".running_mean"], s[name + ".running_var"], s[name + ".weight"], s[name + ".bias"],
                         False, 0.0, 1e-5)
        if self.fault == "bn_scale_dw":     # the value is right, the gradient skips the BN scale
            y = x + (y - x).detach()
        return y

    def dcn(self, x, offset, name, padding=1, dilation=1):
        return torchvision.ops.deform_conv2d(x, offset, self.p[name + ".weight"], self.p.get(name + ".bias"), stride=1,
                                             padding=padding, dilation=dilation)

    # ------------------------------------------------------------------ backbone / FPN / RPN
    def bottleneck(self, x, p, stride, deformable, has_down):
        out = F.relu(self.bn(self.conv(x, p + ".conv1", stride), p + ".bn1"))
        if deformable:
            out = self.dcn(out, self.conv(out, p + ".conv2_offset", 1, 1, 1), p + ".conv2")
        else:
            out = self.conv(out, p + ".conv2", 1, 1, 1)
        out = F.relu(self.bn(out, p + ".bn2"))
        out = self.bn(self.conv(out, p + ".conv3"), p + ".bn3")
        residual = x
        if has_down:
            residual = self.bn(self.conv(x, p + ".downsample.0", stride), p + ".downsample.1")
        return F.relu(out + residual)

    def res_block(self, x, name, blocks, stride, deformable):
        for i in range(max(blocks, 2)):
            x = self.bottleneck(x, "resnet_backbone.%s.layers.%d" % (name, i), stride if i == 0 else 1, deformable, i == 0)
        return x

    def backbone(self, x):
        with torch.set_grad_enabled(self.fault == "res2_trainable"):
            c1 = F.relu(self.bn(self.conv(x, "resnet_backbone.conv1.conv1", 2, 3), "resnet_backbone.conv1.bn1"))
            r2 = self.res_block(F.max_pool2d(c1, 3, 2, 1), "res2", self.depth[0], 1, False)
        if self.fault != "res2_trainable":
            r2 = r2.detach()
        d = self.dconv_from
        r3 = self.res_block(r2, "res3", self.depth[1], 2, d <= 3)
        r4 = self.res_block(r3, "res4", self.depth[2], 2, d <= 4)
        r5 = self.res_block(r4, "res5", self.depth[3], 2, d <= 5)
        return r2, r3, r4, r5

    def fpn(self, r2, r3, r4, r5):
        up = lambda t: F.interpolate(t, scale_factor=2, mode="nearest")     # noqa: E731
        p5_1x1 = self.conv(r5, "fpn.fpn_p5_1x1")
        p4_plus = up(p5_1x1) + self.conv(r4, "fpn.fpn_p4_1x1")
        p3_plus = up(p4_plus) + self.conv(r3, "fpn.fpn_p3_1x1")
        p2_plus = up(p3_plus) + self.conv(r2, "fpn.fpn_p2_1x1")
        p2, p3, p4, p5 = (self.conv(t, "fpn.fpn_p%d" % l, 1, 1) for l, t in ((2, p2_plus), (3, p3_plus), (4, p4_plus),
                                                                             (5, p5_1x1)))
        p6 = F.max_pool2d(p5.detach() if self.fault == "p6_grad" else p5, 1, 2)
        return p2, p3, p4, p5, p6

    def rpn(self, feat):
        x = F.relu(self.conv(feat, "rpn.conv_proposal.0", 1, 1))
        return self.conv(x, "rpn.cls_score"), self.conv(x, "rpn.bbox_pred")

    # ------------------------------------------------------------------ heads
    def fcn_head(self, p2, p3, p4, p5):
        outs = []
        for l, x in enumerate((p2, p3, p4, p5)):
            for i in range(self.fcn_layers):
                p = "fcn_head.fcn_subnet.conv.%d.0" % i
                x = F.relu(self.dcn(x, self.conv(x, p + ".conv_offset", 1, 1, 1), p + ".conv"))
            if self.fault == "fcn_level_detached" and l == 2:
                x = x.detach()
            outs.append(x if l == 0 else F.interpolate(x, None, 2 ** l, mode="bilinear", align_corners=False))
        return self.conv(torch.cat(outs, 1), "fcn_head.score")

    def fpn_roi_align(self, feats, rois, ps):
        r = rois.detach().cpu().numpy().astype(np.float32)
        w, h = r[:, 3] - r[:, 1] + 1, r[:, 4] - r[:, 2] + 1
        lv = np.clip(np.floor(2 + np.log2(np.sqrt(w * h) / 224 + 1e-6)), 0, 3).astype(np.int64)    # fpn_roi_align.py:35-38
        rr = rois.detach().to(feats[0].device, feats[0].dtype)
        parts, order = [], []
        for l in range(4):
            idx = np.where(lv == l)[0]
            if len(idx):
                sel = torch.from_numpy(idx).to(rr.device)
                parts.append(torchvision.ops.roi_align(feats[l], rr[sel], (ps, ps), 1.0 / 2 ** (l + 2), 2, False))
                order.append(idx)
        inv = np.argsort(np.concatenate(order))
        return torch.cat(parts)[torch.from_numpy(inv).to(rr.device)]

    def rcnn(self, feats, rois):
        x = self.fpn_roi_align(feats, rois, 7).flatten(1)
        x = F.relu(F.linear(x, self.p["rcnn.fc6.0.weight"], self.p["rcnn.fc6.0.bias"]))
        x = F.relu(F.linear(x, self.p["rcnn.fc7.0.weight"], self.p["rcnn.fc7.0.bias"]))
        return (F.linear(x, self.p["rcnn.cls_score.weight"], self.p["rcnn.cls_score.bias"]),
                F.linear(x, self.p["rcnn.bbox_pred.weight"], self.p["rcnn.bbox_pred.bias"]))

    def mask_branch(self, feats, rois):
        x = self.fpn_roi_align(feats, rois, 14)
        for i in range(1, 5):
            x = F.relu(self.conv(x, "mask_branch.mask_conv%d.0" % i, 1, 1))
        x = F.relu(F.conv_transpose2d(x, self.p["mask_branch.mask_deconv1.0.weight"],
                                      self.p["mask_branch.mask_deconv1.0.bias"], 2))
        return self.conv(x, "mask_branch.mask_score")

    # ------------------------------------------------------------------ the step
    def forward(self, image, label, inter):
        """image [1,3,H,W]; label: the loader's dict (rpn fields, seg_gt, seg_gt_4x, mask_gt); inter: the product's
        _intermediates.  -> dict of the nine outputs as 0-dim tensors (accuracies as floats)."""
        dev, dt = self.device, self.dtype
        r2, r3, r4, r5 = self.backbone(image.to(dev, dt))
        fpn = self.fpn(r2, r3, r4, r5)
        rpn = [self.rpn(f) for f in fpn]
        rpn_cls = rpn_box = 0
        for (score, pred), s in zip(rpn, STRIDES):
            h, w = score.shape[2:]
            sl = lambda k: label[k % s].to(dev)[:, :, :h, :w]             # noqa: E731
            lab = sl("rpn_labels_fpn%d")
            rpn_cls = rpn_cls + F.binary_cross_entropy_with_logits(score, lab.to(dt), (lab != -1).to(dt),
                                                                   reduction="sum") / self.rpn_batch_size
            rpn_box = rpn_box + TO._smooth_l1(pred, sl("rpn_bbox_targets_fpn%d").to(dt),
                                              sl("rpn_bbox_inside_weights_fpn%d").to(dt),
                                              sl("rpn_bbox_outside_weights_fpn%d").to(dt), 3.0).sum()
        score = self.fcn_head(*fpn[:4])
        up = F.interpolate(score, None, 4, mode="bilinear", align_corners=False)
        fcn_loss = TO.semantic_from_logits(up, label["seg_gt"].to(dev))[0]

        t = inter["proposal_targets"]
        feats = list(fpn[:4])
        cls_score, bbox_pred = self.rcnn(feats, t["rois"])
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
        logits = PO.panoptic_logits(score.cpu().to(dt), pm.cpu().to(dt), gt_rois.detach().cpu().numpy(), cls_idx.cpu().numpy(),
                                    self.num_classes, keep is not None)
        gt = PO.panoptic_gt(label["seg_gt_4x"].cpu().numpy(), label["mask_gt"].cpu().numpy(),
                            None if keep is None else np.asarray(keep), self.num_seg_classes, self.num_classes)
        panoptic_loss, correct, ignored = PO.loss_and_accuracy(logits, gt)
        return {"rpn_cls_loss": rpn_cls, "rpn_bbox_loss": rpn_box, "cls_loss": cls_loss, "bbox_loss": bbox_loss,
                "mask_loss": mask_loss, "fcn_loss": fcn_loss, "panoptic_loss": panoptic_loss.to(dev),
                "rcnn_accuracy": rcnn_acc, "panoptic_accuracy": correct / float(gt.size - ignored)}

    def step(self, image, label, inter):
        """forward + backward of the sum of the seven losses -> (outputs as floats, grads)."""
        out = self.forward(image, label, inter)
        total = sum(out[k] for k in LOSSES)
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
