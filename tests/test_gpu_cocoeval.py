"""Device COCO AP (csrc/cocoeval.cu, DetectionAP) against the COCOeval restatement (tests/coco_oracle.py): precision,
recall, scores and stats bit-identical for 'bbox' and 'segm' on a seeded COCO-like set whose masks come from
ops.im_post_rle on the device, the hand-derived cases, every error flag, repeatability and reset()."""
import functools

import numpy as np
import pytest
import torch

import coco_oracle as CO
from oracle import oracle as O

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
CAT_IDS = [i for i in range(1, 91) if i not in (12, 26, 29, 30, 45, 66, 68, 69, 71, 83)]      # 80 COCO-like ids
CATS = [{"id": c, "name": "c%d" % c} for c in CAT_IDS]


def blob_masks(rng, n):
    yy, xx = np.mgrid[0:28, 0:28].astype(np.float32)
    m = np.zeros((n, 1, 28, 28), np.float32)
    for i in range(n):
        cx, cy, r = rng.uniform(8, 20), rng.uniform(8, 20), rng.uniform(5, 16)
        m[i, 0] = np.clip(1.0 / (1.0 + np.exp(((xx - cx) ** 2 + (yy - cy) ** 2 - r * r) / 18.0)) + rng.normal(0, 0.1, (28, 28)), 0, 1)
    return m


@functools.lru_cache(maxsize=None)
def dataset(seed=7):
    """~60 images at 480x640 and two at 800x1333, 80 categories: crowds, all three area ranges, exact score ties, > 100
    detections of one category in one image, images with detections and no ground truth and the reverse."""
    rng = np.random.default_rng(seed)
    sizes = [(480, 640)] * 60 + [(800, 1333)] * 2
    ids = rng.permutation(np.arange(1000, 1000 + 5 * len(sizes), 5)).tolist()
    out = []
    for i, ((H, W), image_id) in enumerate(zip(sizes, ids)):
        cls_pool = rng.choice(np.arange(1, 81), 4, replace=False)
        gts = []
        ng = 0 if i % 13 == 5 else int(rng.integers(1, 10))
        for _ in range(ng):
            s = float(np.exp(rng.uniform(np.log(8), np.log(min(H, W) * 0.8))))
            w, h = s * rng.uniform(0.6, 1.4), s * rng.uniform(0.6, 1.4)
            x, y = rng.uniform(0, W - w), rng.uniform(0, H - h)
            m = np.zeros((H, W), np.uint8)
            m[int(y):int(y + h), int(x):int(x + w)] = 1
            crowd = int(rng.random() < 0.12)
            enc = O.mask_encode(m)
            gts.append({"category_id": CAT_IDS[int(rng.choice(cls_pool)) - 1], "iscrowd": crowd,
                        "area": float(m.sum()) if rng.random() < 0.8 else float(w * h),
                        "bbox": [float(x), float(y), float(w), float(h)],
                        "segmentation": {"size": [H, W], "counts": enc["counts"].decode()}})
        boxes, cls = [], []
        if i % 11 != 3:
            for g in gts:                                   # near-duplicates of the ground truths
                for _ in range(int(rng.integers(0, 3))):
                    x, y, w, h = g["bbox"]
                    j = rng.normal(0, 0.08 * max(w, h), 4)
                    boxes.append([x + j[0], y + j[1], x + w + j[2], y + h + j[3]])
                    cls.append(CAT_IDS.index(g["category_id"]) + 1 if rng.random() < 0.9 else int(rng.integers(1, 81)))
            for _ in range(int(rng.integers(0, 12))):
                c = rng.uniform([0, 0], [W, H]); s = rng.uniform(4, 300, 2)
                boxes.append([c[0] - s[0] / 2, c[1] - s[1] / 2, c[0] + s[0] / 2, c[1] + s[1] / 2])
                cls.append(int(rng.choice(cls_pool)))
        if i == 7:                                          # > 100 detections of one category in one image
            for _ in range(130):
                c = rng.uniform([0, 0], [W, H]); s = rng.uniform(4, 120, 2)
                boxes.append([c[0] - s[0] / 2, c[1] - s[1] / 2, c[0] + s[0] / 2, c[1] + s[1] / 2])
                cls.append(int(cls_pool[0]))
        n = len(boxes)
        b = np.asarray(boxes, np.float32).reshape(-1, 4)
        b[:, 0::2] = np.clip(b[:, 0::2], 0, W - 1); b[:, 1::2] = np.clip(b[:, 1::2], 0, H - 1)
        scores = (np.round(rng.uniform(0.05, 1.0, n) * 20) / 20).astype(np.float32)        # many exact ties
        out.append(dict(image_id=image_id, H=H, W=W, gts=gts, boxes=b, scores=scores, cls=np.asarray(cls, np.int64),
                        masks=blob_masks(rng, n)))
    return out


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def device_eval(data, iou_type, order=None, ap=None):
    from upsnet_b200 import DetectionAP
    from upsnet_b200 import operators as ops
    ap = ap or DetectionAP(CATS, iou_type)
    for i in (order if order is not None else range(len(data))):
        im = data[i]
        rle = None
        if iou_type == "segm" and len(im["boxes"]) == 0:
            rle = (torch.zeros((0, 16), dtype=torch.int32, device=DEV), torch.zeros(0, dtype=torch.int32, device=DEV))
        elif iou_type == "segm":
            cn, rl, ovf = ops.im_post_rle(t(im["boxes"]), t(im["masks"]), t(im["cls"]), im["H"], im["W"])
            assert int(ovf.item()) == 0
            rle = (cn, rl)
        ap.update(im["image_id"], im["gts"], t(im["boxes"]), t(im["scores"]), t(im["cls"]), rle=rle,
                  im_size=(im["H"], im["W"]))
    return ap, ap.summarize()


@functools.lru_cache(maxsize=None)
def oracle_eval(iou_type):
    data = dataset()
    gts = [dict(g, image_id=im["image_id"]) for im in data for g in im["gts"]]
    images = []
    for im in data:
        segms = None
        if iou_type == "segm":
            imgs = O.im_post_masks(im["boxes"], im["masks"], im["cls"], im["H"], im["W"])
            segms = [O.mask_encode(m) for m in imgs]
        images.append((im["image_id"], im["boxes"], im["scores"], im["cls"], segms))
    return CO.evaluate(gts, images, CAT_IDS, iou_type)


def assert_same(res, E):
    for key in ("precision", "recall", "scores"):
        a, b = res[key], E.eval[key]
        assert a.shape == b.shape
        bad = np.argwhere(a != b)
        assert bad.size == 0, "%s differs at %d entries, first %s: %r vs %r" % (key, len(bad), bad[0], a[tuple(bad[0])], b[tuple(bad[0])])
    assert np.array_equal(res["stats"], E.stats), (res["stats"], E.stats)


@pytest.mark.parametrize("iou_type", ["bbox", "segm"])
def test_device_matches_oracle_bit_identical(iou_type):
    data = dataset()
    order = np.random.default_rng(1).permutation(len(data))          # image ids updated out of order
    _, res = device_eval(data, iou_type, order)
    E = oracle_eval(iou_type)
    assert_same(res, E)
    assert (E.eval["precision"] > 0).any() and (E.eval["precision"] == -1).any()
    from upsnet_b200.evaluation import per_class_ap
    want = per_class_ap(E.eval["precision"])
    for key, v in res["per_class_ap"].items():
        assert np.array_equal([v["mean"]] + v["per_class"], [want[key]["mean"]] + want[key]["per_class"], equal_nan=True)


@pytest.mark.parametrize("iou_type", ["bbox", "segm"])
def test_repeatable_and_reset(iou_type):
    data = dataset()[:20]
    ap, r1 = device_eval(data, iou_type)
    _, r2 = device_eval(data, iou_type)
    ap.reset()
    _, r3 = device_eval(data, iou_type, ap=ap)
    for key in ("precision", "recall", "scores", "stats"):
        assert np.array_equal(r1[key], r2[key]) and np.array_equal(r1[key], r3[key])
    with pytest.raises(ValueError, match="already"):
        ap.update(data[0]["image_id"], [], t(np.zeros((0, 4), np.float32)), t(np.zeros(0, np.float32)),
                  t(np.zeros(0, np.int64)), rle=(torch.zeros((0, 8), dtype=torch.int32, device=DEV),
                                                  torch.zeros(0, dtype=torch.int32, device=DEV)))


def hand_cases():
    """(gts, detections) of the hand-derived cases in test_cocoeval_cpu, on one 200x300 image each, category ids 1, 2."""
    def g(xywh, iscrowd=0):
        return {"category_id": 1, "iscrowd": iscrowd, "bbox": list(map(float, xywh)), "area": float(xywh[2] * xywh[3])}

    def d(x, y, w, h):
        return [x, y, x + w - 1, y + h - 1]
    return [
        ([g((0, 0, 100, 100))], [d(0, 0, 100, 70)], [0.9], [1]),
        ([g((0, 0, 50, 50))], [d(200, 100, 50, 50), d(0, 0, 50, 50)], [0.9, 0.8], [1, 1]),
        ([g((0, 0, 150, 150), 1), g((200, 100, 50, 50))], [d(10, 10, 40, 40), d(200, 100, 50, 50)], [0.95, 0.5], [1, 1]),
        ([g((0, 0, 120, 120))], [d(250, 150, 10, 10), d(0, 0, 120, 120)], [0.9, 0.8], [1, 1]),
        ([g((0, 0, 50, 50)), g((100, 0, 50, 50))], [d(0, 0, 50, 50), d(100, 0, 50, 50)], [0.9, 0.8], [1, 1]),
        ([g((0, 0, 50, 50))], [d(0, 0, 50, 50), d(0, 0, 50, 50)], [0.9, 0.8], [1, 2]),
    ]


@pytest.mark.parametrize("iou_type", ["bbox", "segm"])
@pytest.mark.parametrize("case", range(6))
def test_hand_cases_match_oracle(case, iou_type):
    from upsnet_b200 import DetectionAP
    H, W = 200, 300
    gts, boxes, scores, cls = hand_cases()[case]
    boxes = np.asarray(boxes, np.float32)
    gts = [dict(x) for x in gts]
    segms = []
    for x in gts:                                       # rectangle masks: box and mask IoU agree for these cases
        m = np.zeros((H, W), np.uint8)
        bx, by, bw, bh = (int(v) for v in x["bbox"])
        m[by:by + bh, bx:bx + bw] = 1
        x["segmentation"] = {"size": [H, W], "counts": O.mask_encode(m)["counts"].decode()}
    for b in boxes.astype(int):
        m = np.zeros((H, W), np.uint8)
        m[b[1]:b[3] + 1, b[0]:b[2] + 1] = 1
        segms.append(m)
    ap = DetectionAP([{"id": 1}, {"id": 2}], iou_type)
    rle = None
    if iou_type == "segm":
        cnts = [O.rle_counts(m) for m in segms]
        cap = max(len(c) for c in cnts)
        cn = np.zeros((len(cnts), cap), np.uint32)
        for i, c in enumerate(cnts):
            cn[i, :len(c)] = c
        rle = (t(cn.view(np.int32)), t(np.asarray([len(c) for c in cnts], np.int32)))
    ap.update(1, gts, t(boxes), t(np.float32(scores)), t(np.int64(cls)), rle=rle)
    res = ap.summarize()
    E = CO.evaluate([dict(x, image_id=1) for x in gts],
                    [(1, boxes, np.float32(scores), np.int64(cls), [O.mask_encode(m) for m in segms])], [1, 2], iou_type)
    assert_same(res, E)


def test_error_flags_raise():
    from upsnet_b200 import DetectionAP
    from upsnet_b200._lib import UpsnetError
    from upsnet_b200.evaluation import MAX_AP_DET, MAX_AP_GT, MAX_AP_GT_CAT

    def run(n=1, gts=(), cls=1, iou_type="bbox", cap=1 << 10, gt_size=(20, 30), im_size=(20, 30)):
        ap = DetectionAP([{"id": 1}, {"id": 2}], iou_type, record_capacity=cap)
        b = np.tile(np.float32([[1, 1, 8, 8]]), (n, 1))
        gl = []
        for x in gts:
            m = np.zeros(gt_size, np.uint8); m[1:5, 1:5] = 1
            gl.append(dict(x, segmentation={"size": list(gt_size), "counts": O.mask_encode(m)["counts"].decode()}))
        rle = None
        if iou_type == "segm":
            m = np.zeros(im_size, np.uint8); m[1:9, 1:9] = 1
            c = O.rle_counts(m)
            rle = (t(np.tile(c, (n, 1)).view(np.int32)), t(np.full(n, len(c), np.int32)))
        ap.update(1, gl, t(b), t(np.linspace(0.9, 0.1, n).astype(np.float32)), t(np.full(n, cls, np.int64)), rle=rle,
                  im_size=im_size)
        return ap
    g = {"category_id": 1, "iscrowd": 0, "area": 16.0, "bbox": [1.0, 1.0, 4.0, 4.0]}
    run(gts=[g]).check_errors()
    run(gts=[g], iou_type="segm").check_errors()
    cases = [(dict(n=MAX_AP_DET + 1), "detections in one image"),
             (dict(gts=[g] * (MAX_AP_GT + 1)), "ground truths in one image"),
             (dict(gts=[g] * (MAX_AP_GT_CAT + 1)), "of one category"),
             (dict(cls=3), "class index"),
             (dict(cls=0), "class index"),
             (dict(n=10, cap=5), "record_capacity"),
             (dict(gts=[g], iou_type="segm", gt_size=(30, 20)), "does not cover")]
    for kw, msg in cases:
        with pytest.raises(UpsnetError, match=msg):
            run(**kw).summarize()
    ap = DetectionAP([{"id": 1}], "segm")
    with pytest.raises(ValueError, match="polygon"):
        ap.update(1, [dict(g, segmentation=[[0, 0, 4, 0, 4, 4]])], t(np.zeros((0, 4), np.float32)),
                  t(np.zeros(0, np.float32)), t(np.zeros(0, np.int64)),
                  rle=(torch.zeros((0, 8), dtype=torch.int32, device=DEV), torch.zeros(0, dtype=torch.int32, device=DEV)))
