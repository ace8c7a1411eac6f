"""Plain-torch restatement of the panoptic head of the training forward (models/resnet_upsnet.py:156-179, 250-257 with
unary_logits.py:24-105 and mask_matching.py:37-58), the yardstick of upsnet_b200.training.PanopticLoss.  It builds the
[1,k,h,w] planes explicitly (clarity over speed), runs on the CPU in any float dtype, and takes its gradients from
autograd.  The geometry (windows, bilinear source indices and weights) is float32 in every dtype, as it is in the
reference; only the values are computed in `dtype`.

Also the seeded case generators shared by the CPU tests, the GPU tests, smoke() and scripts/prof_panoptic_loss.py."""
import numpy as np
import torch

F32 = np.float32


def seg_windows(rois, box_scale, h, w):
    """unary_logits.py:89-102: [(y0, y1, x0, x1)] with Python-slice clamping (negative bounds clamped to 0)."""
    b = np.asarray(rois, F32)[:, 1:] * F32(box_scale)
    out = []
    for r in b:
        y0, y1 = int(r[1]), int(np.round(r[3]) + 1)
        x0, x1 = int(r[0]), int(np.round(r[2]) + 1)
        out.append((min(max(y0, 0), h), min(max(y1, 0), h), min(max(x0, 0), w), min(max(x1, 0), w)))
    return out


def resize_matrix(n_out, M, dtype):
    """[n_out, M]: ATen's bilinear rule (align_corners=False) from M samples to n_out, index arithmetic in float32."""
    scale = F32(M) / F32(n_out)
    d = np.arange(n_out, dtype=F32)
    src = np.maximum(scale * (d + F32(0.5)) - F32(0.5), F32(0))
    i0 = np.minimum(src.astype(np.int64), M - 1)
    i1 = i0 + (i0 < M - 1)
    l1 = (src - i0.astype(F32)).astype(F32)
    l0 = (F32(1) - l1).astype(F32)
    R = np.zeros((n_out, M), np.float64)
    np.add.at(R, (np.arange(n_out), i0), l0.astype(np.float64))
    np.add.at(R, (np.arange(n_out), i1), l1.astype(np.float64))
    return torch.from_numpy(R).to(dtype)


def panoptic_logits(fcn, mask_score, rois, cls, num_classes, enable_void, box_scale=0.25):
    """fcn [1,S,h,w], mask_score [k,C,M,M] (C = num_classes or 1) -> [1, num_stuff + k (+1), h, w]."""
    _, S, h, w = fcn.shape
    k, C, M, _ = mask_score.shape
    num_stuff = S - num_classes + 1
    cls = [int(c) for c in cls]
    seg_inst = []
    for (y0, y1, x0, x1), c in zip(seg_windows(rois, box_scale, h, w), cls):
        plane = torch.zeros((h, w), dtype=fcn.dtype)
        if c != 0:
            plane[y0:y1, x0:x1] = fcn[0, num_stuff + c - 1, y0:y1, x0:x1]
        seg_inst.append(plane)
    seg_inst = torch.stack(seg_inst)
    ref = (torch.from_numpy(np.asarray(rois, F32)[:, 1:] * F32(box_scale))).long().tolist()
    mask_inst = []
    for i, (bx0, by0, bx1, by1) in enumerate(ref):
        bw, bh = max(bx1 - bx0 + 1, 1), max(by1 - by0 + 1, 1)
        m = mask_score[i, 0 if C == 1 else cls[i]]
        m = resize_matrix(bh, M, fcn.dtype) @ m @ resize_matrix(bw, M, fcn.dtype).t()
        plane = torch.zeros((h, w), dtype=fcn.dtype)
        x0, x1, y0, y1 = max(bx0, 0), min(bx1 + 1, w), max(by0, 0), min(by1 + 1, h)
        if x1 > x0 and y1 > y0:
            plane[y0:y1, x0:x1] = m[y0 - by0:y1 - by0, x0 - bx0:x1 - bx0]
        mask_inst.append(plane)
    parts = [fcn[0, :num_stuff], seg_inst + torch.stack(mask_inst)]
    if enable_void:
        parts.append((fcn[0, num_stuff:].max(0)[0] - seg_inst.max(0)[0])[None])
    return torch.cat(parts)[None]


def panoptic_gt(seg_gt, mask_gt, keep, S, num_classes):
    """numpy int64 [1,h,w] from seg_gt [1,h,w], mask_gt [G,h,w], keep [k] or None."""
    seg_gt, mask_gt = np.asarray(seg_gt).astype(np.int64), np.asarray(mask_gt).astype(np.int64)
    num_stuff = S - num_classes + 1
    g = np.where((seg_gt <= S - num_classes) | (seg_gt >= 255), seg_gt, -1)
    masks = mask_gt if keep is None else mask_gt[np.asarray(keep)]
    for i in range(masks.shape[0]):
        g[(masks[[i]] != 0) & (masks[[i]] != 255)] = num_stuff + i
    g[g == -1] = 255 if keep is None else num_stuff + masks.shape[0]
    return g


def loss_and_accuracy(logits, gt):
    """-> (loss tensor, correct, ignored): cross-entropy ignoring 255, mean over all pixels; first-arg-max accuracy."""
    gt_t = torch.from_numpy(gt)
    per_pixel = torch.nn.functional.cross_entropy(logits, gt_t, ignore_index=255, reduction="none")
    am = logits.detach().numpy().argmax(1)          # numpy: ties go to the lowest channel
    return per_pixel.mean(), int((am == gt).sum()), int((gt == 255).sum())


def run(case, dtype=torch.float64, grad_out=1.0, C=None):
    """The whole head on one case dict -> dict(loss, accuracy, correct, ignored, logits, gt, d_fcn, d_mask [k,M,M] of
    the selected channels, margin [h,w] = top-1 minus top-2 logit)."""
    fcn = torch.from_numpy(case["fcn"]).to(dtype).requires_grad_(True)
    msk = torch.from_numpy(case["mask_score"] if C != 1 else selected(case)[:, None].numpy()).to(dtype).requires_grad_(True)
    logits = panoptic_logits(fcn, msk, case["rois"], case["cls"], case["num_classes"], case["enable_void"])
    gt = panoptic_gt(case["seg_gt"], case["mask_gt"], case["keep"], fcn.shape[1], case["num_classes"])
    loss, correct, ignored = loss_and_accuracy(logits, gt)
    (loss * grad_out).backward()
    top2 = logits.detach().topk(2, dim=1)[0][0]
    k = msk.shape[0]
    sel = msk.grad[torch.arange(k), torch.from_numpy(case["cls"]) if msk.shape[1] > 1 else 0]
    rest = msk.grad.clone()
    rest[torch.arange(k), torch.from_numpy(case["cls"]) if msk.shape[1] > 1 else 0] = 0
    assert not rest.any()
    return dict(loss=float(loss.detach()), correct=correct, ignored=ignored, accuracy=correct / float(gt.size - ignored),
                logits=logits.detach().numpy(), gt=gt, d_fcn=fcn.grad.numpy(), d_mask=sel.numpy(),
                margin=(top2[0] - top2[1]).numpy())


def selected(case):
    """mask_score[i, cls_i]: float32 [k,M,M]."""
    return torch.from_numpy(case["mask_score"])[torch.arange(len(case["cls"])), torch.from_numpy(case["cls"])]


# ------------------------------------------------------------------------------------------------ case generators
def make_case(seed, S, num_classes, h, w, G, k=None, enable_void=True):
    """One image at quarter resolution h x w (network input 4h x 4w) with G ground-truth objects; with enable_void, k of
    them are kept in a permuted order (k < G), else all G.  The first objects are the hand-placed ones, as far as G
    allows: 0 reaches past the right / bottom edge of the image, 1 is smaller than one quarter-resolution pixel, 2 is
    wider than mask_size quarter-pixels, 3 narrower, 4 and 5 share a class and overlap (boxes and masks), 6 has class 0.
    mask_gt holds 255 in places, seg_gt holds 255 and thing-class labels no mask covers."""
    rng = np.random.default_rng(seed)
    H, W = 4 * h, 4 * w
    num_stuff = S - num_classes + 1
    c = np.stack([rng.uniform(0, W, G), rng.uniform(0, H, G)], 1)
    s = np.exp(rng.uniform(np.log(12), np.log(min(H, W) * 0.9), (G, 2)))
    boxes = np.concatenate([c - s / 2, c + s / 2], 1)
    cls = rng.integers(1, num_classes, G).astype(np.int64)
    hand = [[W - 50.3, H - 41.2, W + 30.5, H + 17.7], [21.3, 33.1, 22.9, 34.2], [8.6, 10.2, min(8.6 + 130.5, W - 6.5), 47.9],
            [60.4, 20.5, 60.4 + 41.3, 20.5 + 37.6], [30.2, 40.1, 75.5, 88.6], [48.7, 52.3, 92.4, 93.9], [5.1, 60.2, 44.4, 90.3]]
    for i, b in enumerate(hand[:G]):
        boxes[i] = b
    if G > 5:
        cls[5] = cls[4]
    if G > 6:
        cls[6] = 0
    boxes[:, 0::2] = np.clip(boxes[:, 0::2], 0, None)
    boxes[:, 1::2] = np.clip(boxes[:, 1::2], 0, None)
    boxes[len(hand):, 0::2] = np.clip(boxes[len(hand):, 0::2], 0, W - 1)
    boxes[len(hand):, 1::2] = np.clip(boxes[len(hand):, 1::2], 0, H - 1)
    boxes = boxes.astype(F32)
    # ground-truth masks: an ellipse in each box at quarter resolution, a stripe of 255 through some of them
    yy, xx = np.mgrid[0:h, 0:w]
    mask_gt = np.zeros((G, h, w), np.uint8)
    for i, (x1, y1, x2, y2) in enumerate(boxes / 4):
        cx, cy, rx, ry = (x1 + x2) / 2, (y1 + y2) / 2, max((x2 - x1) / 2, 0.6), max((y2 - y1) / 2, 0.6)
        mask_gt[i] = ((xx + 0.5 - cx) / rx) ** 2 + ((yy + 0.5 - cy) / ry) ** 2 <= 1
        if i % 3 == 2:
            mask_gt[i, int(cy) % h, :] = np.where(mask_gt[i, int(cy) % h, :], 255, 0)
    # semantic labels: blocky stuff, thing labels under the masks and in a few places no mask covers, a band of 255
    seg_gt = np.kron(rng.integers(0, num_stuff, (-(-h // 8), -(-w // 8))), np.ones((8, 8), np.int64))[:h, :w].astype(np.int64)
    for i in range(G):
        if cls[i] > 0:
            seg_gt[mask_gt[i] == 1] = num_stuff + cls[i] - 1
    seg_gt[h // 2:h // 2 + 2, : w // 3] = num_stuff + int(rng.integers(0, num_classes - 1))
    seg_gt[: max(h // 12, 1)] = 255
    seg_gt[:, w - 1] = 255
    if enable_void:
        k = k if k is not None else max(G - 2, 1)
        assert 0 < k < G or G == 1
        first = list(range(min(len(hand), k)))
        rest = [i for i in rng.permutation(G).tolist() if i not in first][:k - len(first)]
        keep = np.asarray(first + rest, np.int64)[rng.permutation(k)]
        rois_cls = cls[keep]
        kept_boxes = boxes[keep]
    else:
        keep, rois_cls, kept_boxes, k = None, cls, boxes, G
    rois = np.concatenate([np.zeros((k, 1), F32), kept_boxes], 1).astype(F32)
    fcn = (rng.standard_normal((1, S, h, w)) * 2).astype(F32)
    mask_score = (rng.standard_normal((k, num_classes, 28, 28)) * 2).astype(F32)
    return dict(fcn=fcn, mask_score=mask_score, rois=rois, cls=rois_cls.astype(np.int64), seg_gt=seg_gt[None],
                mask_gt=mask_gt, keep=keep, num_classes=num_classes, enable_void=enable_void)


# name -> (seed, S, num_classes, h, w, G, k, enable_void)
SMALL = {"cityscapes_void": (11, 19, 9, 32, 48, 10, 8, True), "coco_void": (12, 133, 81, 24, 40, 9, 7, True),
         "no_void": (13, 19, 9, 24, 40, 8, None, False)}
FULL = {"cityscapes": (21, 19, 9, 256, 512, 40, 35, True), "coco_k63": (22, 133, 81, 200, 336, 70, 63, True),
        "coco_k10": (23, 133, 81, 200, 336, 12, 10, True)}
SMOKE = (7, 19, 9, 24, 40, 5, 3, True)


def digest(a):
    """sha256 of an array's bytes (C order), as the fixture stores it for the one large random input."""
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def case(spec):
    seed, S, nc, h, w, G, k, void = spec
    return make_case(seed, S, nc, h, w, G, k, void)
