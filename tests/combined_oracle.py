"""numpy restatement of the combined panoptic result (dataset/base_dataset.py:373-449 get_combined_pan_result +
_merge_pred_single_core) for ONE image, with the merge order of rule 2 of DESIGN.md section 3 fixed (the reference's
default argsort leaves exact score ties unordered), the uint8 wraps of the reference spelled out, and the float32 keep
test of numpy >= 2.  Shared by the fixture generator (tests/golden/make_reference_combined.py) and the tests: the seeded
1024x2048 image is rebuilt here, so only its digest is stored."""
import hashlib

import numpy as np

from oracle import oracle as O


def merge_order(scores, cls_inds, num_classes):
    """Detections (input indices) in the order the merge takes them: descending score, ties by the later position in
    im_post's class-ascending concatenation, i.e. (score desc, class desc, index desc).  np.lexsort puts NaN after
    every number, as np.argsort does, and compares -0 and +0 equal.  Classes outside [1, num_classes) are dropped (im_post
    never emits them)."""
    s = np.asarray(scores, np.float32).reshape(-1)
    c = np.asarray(cls_inds, np.int64).reshape(-1)
    order = np.lexsort((np.arange(s.size), c, s))[::-1]
    return [int(d) for d in order if 1 <= c[d] < num_classes]


def combined_pan_result(sem, scores, cls_inds, runs, num_seg_classes, num_classes, score_threshold=0.6,
                        fraction_threshold=0.7, stuff_area_limit=4 * 64 * 64):
    """sem [H,W] ints (wrapped to uint8 like the restored map); scores / cls_inds [n]; runs: n uncompressed COCO run-length
    arrays of H x W masks.  -> uint8 [H,W,3] (class, instance number, 0)."""
    sem = np.asarray(sem).astype(np.uint8)
    H, W = sem.shape
    id_last = num_seg_classes - num_classes
    thr_s, thr_f = np.float32(score_threshold), np.float32(fraction_threshold)
    scores = np.asarray(scores, np.float32).reshape(-1)
    cls_inds = np.asarray(cls_inds, np.int64).reshape(-1)
    ins = np.zeros((H, W), np.uint8)                     # instance number; 0 = not claimed
    ins_cls = np.zeros((H, W), np.int64)
    count = np.zeros(max(num_classes - 1, 1), np.int64)  # kept instances per class (the uint32 idx_ins_array)
    for d in merge_order(scores, cls_inds, num_classes):
        if scores[d] < thr_s:
            continue
        r = np.asarray(runs[d], np.int64)
        assert int(r.sum()) == H * W, "RLE does not cover the semantic map"
        m = O.rle_decode(r, H, W).astype(bool)
        free = m & (ins == 0)
        area, remain = int(m.sum()), int(free.sum())
        # both sums are float32 in the reference, and numpy >= 2 compares the float32 ratio with float32(threshold)
        if area == 0 or np.float32(remain) / np.float32(area) < thr_f:
            continue
        c = int(cls_inds[d])
        count[c - 1] += 1
        ins[free] = count[c - 1] % 256                   # stored into uint8: the 256th instance writes 0
        ins_cls[free] = c
    hist = np.bincount(sem.ravel(), minlength=256)
    small = (np.arange(256) <= id_last) & (hist < stuff_area_limit)
    c0 = np.where(small[sem], 255, sem.astype(np.int64))
    c0 = np.where((c0 > id_last) & (ins == 0), 255, c0)
    c0 = np.where(ins != 0, (ins_cls + id_last) % 256, c0)
    out = np.zeros((H, W, 3), np.uint8)
    out[..., 0] = c0
    out[..., 1] = ins
    return out


def pack_runs(runs):
    """n run-length arrays -> (counts uint32 [max(n,1), cap], run_len int32 [max(n,1)]) in im_post_rle's layout."""
    cap = max([len(r) for r in runs] + [1])
    cn = np.zeros((max(len(runs), 1), cap), np.uint32)
    rl = np.zeros(max(len(runs), 1), np.int32)
    for d, r in enumerate(runs):
        cn[d, :len(r)] = r
        rl[d] = len(r)
    return cn, rl


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def blob_mask(rng, H, W, cy, cx, ry, rx):
    """An elliptical mask with a ragged border, clipped to the image."""
    yy, xx = np.ogrid[0:H, 0:W]
    d = ((yy - cy) / max(ry, 1.0)) ** 2 + ((xx - cx) / max(rx, 1.0)) ** 2
    return (d < 1.0 + 0.15 * np.sin(yy * 0.37 + xx * 0.23 + rng.uniform(0, 6))).astype(np.uint8)


def semantic_map(rng, H, W, num_seg_classes, block=16):
    """Blocks of random classes (plus a little 255 void), with a few classes kept rare so the stuff limit bites."""
    hb, wb = (H + block - 1) // block, (W + block - 1) // block
    sem = np.kron(rng.integers(0, num_seg_classes, (hb, wb)), np.ones((block, block), np.int64))[:H, :W]
    sem[np.kron(rng.random((hb, wb)) < 0.03, np.ones((block, block), bool))[:H, :W]] = 255
    return sem.astype(np.uint8)


def random_detections(rng, H, W, n, num_classes, score_lo=0.3):
    """n detections in engine order (classes mixed): scores, classes and the run lengths of blob masks."""
    scores = rng.uniform(score_lo, 1.0, n).astype(np.float32)
    cls = rng.integers(1, num_classes, n).astype(np.int64)
    runs = []
    for _ in range(n):
        cy, cx = rng.uniform(0, H), rng.uniform(0, W)
        ry, rx = rng.uniform(2, H / 6), rng.uniform(2, W / 6)
        runs.append(O.rle_counts(blob_mask(rng, H, W, cy, cx, ry, rx)))
    return scores, cls, runs


LARGE = dict(H=1024, W=2048, n=100, num_seg_classes=19, num_classes=9, seed=2048)


def large_case():
    """The seeded 1024x2048 Cityscapes-sized image with about 100 detections."""
    rng = np.random.default_rng(LARGE["seed"])
    H, W = LARGE["H"], LARGE["W"]
    sem = semantic_map(rng, H, W, LARGE["num_seg_classes"], block=64)
    scores, cls, runs = random_detections(rng, H, W, LARGE["n"], LARGE["num_classes"])
    return sem, scores, cls, runs
