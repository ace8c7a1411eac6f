"""Test infrastructure: a numpy restatement of the reference's semantic-segmentation evaluation (evaluate_ssegs +
write_segmentation_result, dataset/cityscapes.py:445-514 / coco.py:225-293, and get_confusion_matrix,
base_dataset.py:806-824), of Pillow's NEAREST resize rule and of the test script's restore step composed with it.  The
oracle of record for csrc/sseg.cu on the GPU machine, which has neither the reference nor, necessarily, PIL;
tests/golden/make_reference_sseg.py pins it to the reference's own code (tests/test_sseg_cpu.py).  The product package
never imports this module."""
import numpy as np

import pq_oracle as P


def pil_index(n_in, n_out):
    """Source indices of PIL Image.resize(NEAREST) along one axis (libImaging/Geometry.c ImagingScaleAffine): xo starts at
    a / 2 and grows by a = n_in / n_out per output pixel, each step rounded to double; the index is (int) xo."""
    a = n_in / n_out
    xo = a * 0.5
    out = np.empty(n_out, np.int64)
    for i in range(n_out):
        out[i] = int(xo)
        xo += a
    return out


def pil_resize(img, H, W):
    """img [h, w] -> [H, W] by Pillow's NEAREST rule (the identity when the sizes are equal)."""
    return img[pil_index(img.shape[0], H)][:, pil_index(img.shape[1], W)]


def prediction_at_gt(pred, gt_shape, im_info=None):
    """The prediction as evaluate_ssegs compares it with the ground truth: with im_info, first the test script's crop +
    cv2 restore (pq_oracle.label_restore); then np.uint8 (values wrap mod 256) and Pillow's resize to the gt size."""
    p = np.asarray(pred)
    if im_info is not None:
        p = P.label_restore(p, im_info)
    p = p.reshape(p.shape[-2:]).astype(np.uint8)
    return pil_resize(p, *gt_shape)


def confusion(pred, gt, num_classes, im_info=None):
    """float64 [C, C] of one image: gt == 255 ignored, bin (gt * C + pred) in float32 then int32, bins >= C*C dropped."""
    gt = np.asarray(gt)
    p = prediction_at_gt(pred, gt.shape, im_info)
    keep = gt != 255
    f = (gt[keep].astype(np.float32) * num_classes + p[keep]).astype(np.int32)
    f = f[f < num_classes * num_classes]
    return np.bincount(f, minlength=num_classes * num_classes).reshape(num_classes, num_classes).astype(np.float64)


def summarize(confusion_matrix):
    """evaluate_ssegs's evaluation_results from the accumulated matrix."""
    pos = confusion_matrix.sum(1)
    res = confusion_matrix.sum(0)
    tp = np.diag(confusion_matrix)
    IU_array = (tp / np.maximum(1.0, pos + res - tp))
    return {'meanIU': IU_array.mean(), 'IU_array': IU_array, 'confusion_matrix': confusion_matrix}


def log_lines(results):
    """The '%.5f' lines evaluate_ssegs logs for IU_array and meanIU."""
    return ['%.5f' % v for v in results['IU_array']] + ['meanIU:%.5f' % results['meanIU']]


def _hash(y, x, k):
    v = (y * 73856093) ^ (x * 19349663) ^ ((k + 1) * 83492791)
    v = (v ^ (v >> 13)) * 0x5bd1e995
    return (v ^ (v >> 15)) & 0x7fffffff


def synthetic_case(k, H, W, num_classes, pred_hw=None):
    """Deterministic (pred int64 [h, w], gt uint8 [H, W]) for case k, rebuilt from an integer hash (no RNG stream):
    37x53 label blocks with about 1/(C+2) of them ignored (255) and as many carrying an out-of-range class; a
    prediction made of the same blocks offset by (11, 17) px (classes C and C+1 alias), with 5 % per-pixel noise in
    [-40, 300) (wrapping)."""
    ph, pw = pred_hw or (H, W)
    y, x = np.arange(H, dtype=np.int64)[:, None], np.arange(W, dtype=np.int64)[None, :]
    b = _hash(y // 37, x // 53, k) % (num_classes + 2)
    gt = np.where(b == num_classes, 255, np.where(b == num_classes + 1, min(num_classes + 7, 254), b)).astype(np.uint8)
    y, x = np.arange(ph, dtype=np.int64)[:, None], np.arange(pw, dtype=np.int64)[None, :]
    pred = _hash((y * H // ph + 11) // 37, (x * W // pw + 17) // 53, k) % (num_classes + 2)
    noise = _hash(y, x, k + 1000)
    return np.where(noise % 20 == 0, noise // 20 % 340 - 40, pred), gt
