"""Plain-torch restatements of the semantic, RPN and Mask R-CNN training losses (upsnet_b200.training.SemanticLoss,
RPNLoss, MaskRCNNLoss), in any float dtype (float64 in the tests), gradients by autograd, and the seeded case generators
the fixtures, tests, smoke() and scripts/prof_train_losses.py share.

* semantic: models/fcn.py:101 + models/resnet_upsnet.py:131, CrossEntropyLoss(ignore_index=255)(F.interpolate(
  fcn_score, None, 4, mode='bilinear', align_corners=False), seg_gt).  A label that is neither 255 nor a channel (torch
  asserts on it) is restated as ignored, and counted apart.
* rpn: models/rpn.py:60-92 (with_fpn): per level the [:, :, :h, :w] slices, BCE-with-logits (weight label != -1, sum /
  rpn_batch_size) and smooth-L1 (sigma 3, inside / outside weights, sum / batch), summed over the levels.
* mask_rcnn: models/rcnn.py:159-197: cross-entropy (ignore -1), smooth-L1 (sigma 1, sum / R), rcnn_accuracy and the mask
  loss / (sum of weights + 1e-10)."""
import hashlib

import numpy as np
import torch
import torch.nn.functional as F

STRIDES = (4, 8, 16, 32, 64)


def digest(a):
    a = np.ascontiguousarray(a)
    return hashlib.sha256(str(a.dtype).encode() + str(a.shape).encode() + a.tobytes()).hexdigest()


# ------------------------------------------------------------------------------------------------
# semantic loss
# ------------------------------------------------------------------------------------------------
def semantic_case(seed, S, h, w, pad=(0, 0), ignore=0.1, invalid=0.0):
    """fcn_score float32 [1,S,h,w]; seg_gt uint8 [1,4h,4w]: random labels, a fraction `ignore` of 255, the last pad[0]
    rows and pad[1] columns 255 (the padding of the blob), and a fraction `invalid` of labels in S..254."""
    rng = np.random.default_rng(seed)
    fcn = (rng.standard_normal((1, S, h, w)) * 3).astype(np.float32)
    seg = rng.integers(0, S, (1, 4 * h, 4 * w)).astype(np.uint8)
    seg[rng.random(seg.shape) < ignore] = 255
    if invalid:
        bad = rng.random(seg.shape) < invalid
        seg[bad] = rng.integers(S, 255, int(bad.sum()))
    if pad[0]:
        seg[:, 4 * h - pad[0]:] = 255
    if pad[1]:
        seg[:, :, 4 * w - pad[1]:] = 255
    return dict(fcn=fcn, seg_gt=seg)


def semantic_from_logits(logits, seg_gt):
    """The cross-entropy part on given [1,S,H,W] logits (tensor); -> (loss tensor, N, invalid)."""
    S = logits.shape[1]
    seg = torch.as_tensor(np.asarray(seg_gt)).long() if not torch.is_tensor(seg_gt) else seg_gt.long()
    seg = seg.to(logits.device)
    bad = (seg != 255) & ((seg < 0) | (seg >= S))
    seg = torch.where(bad, torch.full_like(seg, 255), seg)
    loss = F.cross_entropy(logits, seg, ignore_index=255)
    return loss, int((seg != 255).sum()), int(bad.sum())


def semantic(c, dtype=torch.float64, device="cpu"):
    """-> dict(loss, n, invalid, d_fcn) for a semantic_case dict (fcn, seg_gt)."""
    x = torch.from_numpy(c["fcn"]).to(device, dtype).requires_grad_(True)
    up = F.interpolate(x, None, 4, mode="bilinear", align_corners=False)
    loss, n, bad = semantic_from_logits(up, c["seg_gt"])
    loss.backward()
    return dict(loss=float(loss.detach()), n=n, invalid=bad, d_fcn=x.grad.cpu().numpy())


# ------------------------------------------------------------------------------------------------
# RPN loss
# ------------------------------------------------------------------------------------------------
def rpn_case(seed, im_h, im_w, field, A=3, fg=0.02, bg=0.2):
    """Score and box maps of an im_h x im_w image (level size ceil(im / stride)) and a label dict on square fields of
    ceil(field / stride), the layout RPNTargets writes: labels -1 / 0 / 1, inside weights 1 on fg anchors, outside
    weights 1 / (fg + bg) on labelled anchors.  numpy arrays."""
    rng = np.random.default_rng(seed)
    scores, preds, label = [], [], {}
    for s in STRIDES:
        h, w, Fs = -(-im_h // s), -(-im_w // s), -(-field // s)
        scores.append((rng.standard_normal((1, A, h, w)) * 2).astype(np.float32))
        preds.append((rng.standard_normal((1, 4 * A, h, w)) * 0.3).astype(np.float32))
        u = rng.random((1, A, Fs, Fs))
        lab = np.where(u < fg, 1, np.where(u < fg + bg, 0, -1)).astype(np.int64)
        label["rpn_labels_fpn%d" % s] = lab
        label["rpn_bbox_targets_fpn%d" % s] = (rng.standard_normal((1, 4 * A, Fs, Fs)) * 0.3).astype(np.float32)
        fg4 = np.repeat(lab == 1, 4, axis=1)
        label["rpn_bbox_inside_weights_fpn%d" % s] = fg4.astype(np.float32)
        label["rpn_bbox_outside_weights_fpn%d" % s] = np.repeat(lab != -1, 4, axis=1).astype(np.float32) / np.float32(
            max(int((lab != -1).sum()), 1))
    return dict(scores=scores, preds=preds, label=label)


def _smooth_l1(pred, target, iw, ow, sigma):
    s2 = sigma ** 2
    d = iw * (pred - target)
    a = d.abs()
    sign = (a < 1.0 / s2).to(pred.dtype)
    return (d ** 2 * (s2 / 2.0) * sign + (a - 0.5 / s2) * (1.0 - sign)) * ow


def rpn(c, batch, dtype=torch.float64, device="cpu"):
    """-> dict(cls_loss, bbox_loss, d_scores [per level], d_preds [per level])."""
    xs = [torch.from_numpy(a).to(device, dtype).requires_grad_(True) for a in c["scores"]]
    ps = [torch.from_numpy(a).to(device, dtype).requires_grad_(True) for a in c["preds"]]
    cls_l, box_l = 0, 0
    for x, p, s in zip(xs, ps, STRIDES):
        h, w = x.shape[2:]
        sl = lambda k: torch.from_numpy(c["label"][k % s]).to(device)[:, :, :h, :w]  # noqa: E731
        lab = sl("rpn_labels_fpn%d")
        cls_l = cls_l + F.binary_cross_entropy_with_logits(x, lab.to(dtype), (lab != -1).to(dtype), reduction="sum") / batch
        box = _smooth_l1(p, sl("rpn_bbox_targets_fpn%d").to(dtype), sl("rpn_bbox_inside_weights_fpn%d").to(dtype),
                         sl("rpn_bbox_outside_weights_fpn%d").to(dtype), 3.0)
        box_l = box_l + box.sum() / p.shape[0]
    (cls_l + box_l).backward()
    return dict(cls_loss=float(cls_l.detach()), bbox_loss=float(box_l.detach()), d_scores=[x.grad.cpu().numpy() for x in xs],
                d_preds=[p.grad.cpu().numpy() for p in ps])


# ------------------------------------------------------------------------------------------------
# Mask R-CNN loss
# ------------------------------------------------------------------------------------------------
def mask_rcnn_case(seed, R, K, n, M=28, ignore=0.0, all_ignored_mask=False):
    """cls_score [R,K], labels in 0..K-1 (about a quarter fg) with a fraction `ignore` of -1, the box tensors [R,4K]
    (class-specific targets of fg rows, as ProposalTargets writes), mask_score [n,K,M,M] and mask_target [n,K*M*M]
    (0 / 1 in the row's class channel, -1 elsewhere, or -1 everywhere).  numpy arrays."""
    rng = np.random.default_rng(seed)
    cls_score = (rng.standard_normal((R, K)) * 2).astype(np.float32)
    label = np.where(rng.random(R) < 0.25, rng.integers(1, K, R), 0).astype(np.int64)
    label[:n] = rng.integers(1, K, n)
    label[rng.random(R) < ignore] = -1
    pred = (rng.standard_normal((R, 4 * K)) * 0.8).astype(np.float32)
    tgt = np.zeros((R, 4 * K), np.float32)
    iw = np.zeros((R, 4 * K), np.float32)
    for r in np.flatnonzero(label > 0):
        c = label[r]
        tgt[r, 4 * c:4 * c + 4] = rng.standard_normal(4) * 0.8
        iw[r, 4 * c:4 * c + 4] = 1
    ow = iw.copy()
    mask_score = (rng.standard_normal((n, K, M, M)) * 3).astype(np.float32)
    mt = np.full((n, K, M, M), -1, np.float32)
    if not all_ignored_mask:
        for i in range(n):
            mt[i, max(int(label[i]), 0)] = rng.random((M, M)) < 0.4
    return dict(cls_score=cls_score, bbox_pred=pred, mask_score=mask_score, cls_label=label, bbox_target=tgt,
                bbox_inside_weight=iw, bbox_outside_weight=ow, mask_target=mt.reshape(n, K * M * M))


NAMES = ("cls_score", "bbox_pred", "mask_score", "cls_label", "bbox_target", "bbox_inside_weight", "bbox_outside_weight",
         "mask_target")


def mask_rcnn(c, dtype=torch.float64, device="cpu"):
    """-> dict(cls_loss, bbox_loss, mask_loss, accuracy, valid, ignored, matches, mask_weight, d_cls, d_bbox, d_mask).
    Labels outside -1..K-1 count as neither valid nor ignored."""
    x = torch.from_numpy(c["cls_score"]).to(device, dtype).requires_grad_(True)
    p = torch.from_numpy(c["bbox_pred"]).to(device, dtype).requires_grad_(True)
    m = torch.from_numpy(c["mask_score"]).to(device, dtype).requires_grad_(True)
    lab = torch.from_numpy(c["cls_label"]).to(device).long()
    R, K = x.shape
    bad = (lab != -1) & ((lab < 0) | (lab >= K))
    lab_ce = torch.where(bad, torch.full_like(lab, -1), lab)
    cls_loss = F.cross_entropy(x, lab_ce, ignore_index=-1)
    box = _smooth_l1(p, *(torch.from_numpy(c[k]).to(device, dtype) for k in ("bbox_target", "bbox_inside_weight",
                                                                       "bbox_outside_weight")), 1.0)
    bbox_loss = box.sum() / box.shape[0]
    pred = x.detach().argmax(1)
    ignore = int((lab == -1).sum())
    matches = int((pred == lab).sum())
    acc = (matches - ignore) / float(R - ignore)
    t = torch.from_numpy(c["mask_target"]).to(device, dtype).view(m.shape)
    wgt = (t != -1).to(dtype)
    b = (m >= 0).to(dtype)
    term = -m * (t - b) + torch.log1p(torch.exp(m - 2 * m * b))
    mask_loss = (term * wgt).sum() / (wgt.sum() + 1e-10)
    (cls_loss + bbox_loss + mask_loss).backward()
    return dict(cls_loss=float(cls_loss.detach()), bbox_loss=float(bbox_loss.detach()), mask_loss=float(mask_loss.detach()), accuracy=acc,
                valid=int(((lab >= 0) & (lab < K)).sum()), ignored=ignore, matches=matches, mask_weight=int(wgt.sum()),
                d_cls=x.grad.cpu().numpy(), d_bbox=p.grad.cpu().numpy(), d_mask=m.grad.cpu().numpy())


# the small cases of the fixtures (reference_train_losses.npz) and smoke()
SEM_SMALL = {"cityscapes": (3, 19, 12, 20, (6, 10), 0.1, 0.0), "coco_s133": (4, 133, 9, 7, (0, 3), 0.2, 0.0)}
RPN_SMALL = {"fields_larger": (5, 90, 130, 160), "same_size": (6, 64, 64, 64)}
MRCNN_SMALL = {"coco": (7, 32, 81, 6, 28, 0.0, False), "ignored_rows": (8, 24, 9, 4, 28, 0.3, False),
               "no_mask_target": (9, 16, 9, 3, 28, 0.0, True)}
