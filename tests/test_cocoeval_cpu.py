"""The COCOeval restatement (tests/coco_oracle.py) against hand-derived answers that do not depend on it, against the
reference-executed fixtures (tests/golden/reference_cocoeval.npz), and against real pycocotools where it is installed;
plus the host halves of DetectionAP (summarize, per-class slicing, RLE parsing)."""
import os

import numpy as np
import pytest

import coco_oracle as CO
from oracle import oracle as O
from upsnet_b200 import evaluation as EV
from upsnet_b200 import operators as ops

GOLD_PATH = os.path.join(os.path.dirname(__file__), "golden", "reference_cocoeval.npz")


def box_gt(image_id, cat, xywh, area=None, iscrowd=0, id_=None):
    a = {"image_id": image_id, "category_id": cat, "iscrowd": iscrowd, "bbox": list(map(float, xywh)),
         "area": float(xywh[2] * xywh[3] if area is None else area)}
    if id_ is not None:
        a["id"] = id_
    return a


def det(image_id, boxes, scores, cls):
    return (image_id, np.asarray(boxes, np.float32).reshape(-1, 4), np.asarray(scores, np.float32),
            np.asarray(cls, np.int64), None)


def xyxy(x, y, w, h):            # the detection box whose xyxy_to_xywh is (x, y, w, h)
    return [x, y, x + w - 1, y + h - 1]


P1 = 1 / (1 + np.spacing(1))     # precision of one tp and no fp: pr = tp / (fp + tp + np.spacing(1)) is just below 1


def ap(E, t=slice(None), k=0, a=0, m=2):
    p = E.eval["precision"][t, :, k, a, m]
    return float(np.mean(p[p > -1]))


def test_iou_07_gives_ap_half():
    # gt 100x100, detection 100x70 inside it: IoU 0.7 exactly -> true positive at t <= 0.7 (5 of 10 thresholds)
    E = CO.evaluate([box_gt(1, 1, (0, 0, 100, 100))], [det(1, [xyxy(0, 0, 100, 70)], [0.9], [1])], [1], "bbox")
    assert E.ious[1, 1][0, 0] == 0.7
    assert np.all(E.eval["precision"][:5, :, 0, 0, 2] == P1) and np.all(E.eval["precision"][5:, :, 0, 0, 2] == 0)
    assert ap(E) == pytest.approx(0.5, rel=1e-15)
    assert E.stats[1] == np.mean(np.full(101, P1)) and E.stats[2] == 0.0


def test_false_positive_ahead_of_true_positive():
    # fp at 0.9, tp at 0.8: pr = [0, 1/2], envelope [1/2, 1/2]; recall 1 reached at the 2nd detection -> AP 0.5
    E = CO.evaluate([box_gt(1, 1, (0, 0, 50, 50))],
                    [det(1, [xyxy(200, 200, 50, 50), xyxy(0, 0, 50, 50)], [0.9, 0.8], [1, 1])], [1], "bbox")
    assert np.all(E.eval["precision"][:, :, 0, 0, 2] == 0.5)
    assert ap(E) == 0.5


def test_detection_on_crowd_is_neither_tp_nor_fp():
    # a crowd region and one regular gt; the detection on the crowd is ignored, the one on the gt is a tp: AP 1
    gts = [box_gt(1, 1, (0, 0, 200, 200), iscrowd=1), box_gt(1, 1, (300, 300, 50, 50))]
    E = CO.evaluate(gts, [det(1, [xyxy(10, 10, 40, 40), xyxy(300, 300, 50, 50)], [0.95, 0.5], [1, 1])], [1], "bbox")
    e = E.evalImgs[0]
    assert e["dtIgnore"][:, 0].all() and not e["dtIgnore"][:, 1].any() and e["dtMatches"][:, 1].all()
    assert ap(E) == P1
    # crowd IoU is inter / area(dt): 1600 / 1600
    assert E.ious[1, 1][0, 0] == 1.0


def test_unmatched_small_detection_ignored_in_large_range():
    # a large gt found; an extra small detection with a higher score is a fp in 'all' but ignored in 'large'
    gts = [box_gt(1, 1, (0, 0, 120, 120))]
    E = CO.evaluate(gts, [det(1, [xyxy(500, 500, 10, 10), xyxy(0, 0, 120, 120)], [0.9, 0.8], [1, 1])], [1], "bbox")
    assert ap(E, a=0) == 0.5 and ap(E, a=3) == P1
    assert E.evalImgs[3 * 1]["dtIgnore"][:, 0].all()


def test_max_dets_1_vs_10_recall():
    # two gts, two matching detections: maxDets 1 finds one of them (recall 0.5), 10 finds both (1.0)
    gts = [box_gt(1, 1, (0, 0, 50, 50)), box_gt(1, 1, (100, 0, 50, 50))]
    E = CO.evaluate(gts, [det(1, [xyxy(0, 0, 50, 50), xyxy(100, 0, 50, 50)], [0.9, 0.8], [1, 1])], [1], "bbox")
    assert np.all(E.eval["recall"][:, 0, 0, 0] == 0.5) and np.all(E.eval["recall"][:, 0, 0, 1] == 1.0)
    assert E.stats[6] == 0.5 and E.stats[7] == 1.0


def test_category_without_ground_truth_is_minus_one():
    E = CO.evaluate([box_gt(1, 1, (0, 0, 50, 50))],
                    [det(1, [xyxy(0, 0, 50, 50), xyxy(0, 0, 50, 50)], [0.9, 0.8], [1, 2])], [1, 2], "bbox")
    assert np.all(E.eval["precision"][:, :, 1] == -1) and np.all(E.eval["recall"][:, 1] == -1)
    assert np.all(E.eval["scores"][:, :, 1] == -1)
    assert ap(E) == P1


def test_segm_iou_and_crowd_area():
    H, W = 40, 30
    g = np.zeros((H, W), np.uint8); g[5:25, 3:13] = 1                  # 200 px
    d = np.zeros((H, W), np.uint8); d[15:35, 3:13] = 1                 # 200 px, 100 shared
    gt = {"image_id": 1, "category_id": 1, "iscrowd": 0, "area": 200.0, "segmentation": O.mask_encode(g)}
    E = CO.evaluate([gt], [(1, np.zeros((1, 4), np.float32), np.float32([0.5]), np.int64([1]), [O.mask_encode(d)])],
                    [1], "segm")
    assert E.ious[1, 1][0, 0] == 100 / 300
    crowd = dict(gt, iscrowd=1)
    E = CO.evaluate([crowd], [(1, np.zeros((1, 4), np.float32), np.float32([0.5]), np.int64([1]), [O.mask_encode(d)])],
                    [1], "segm")
    assert E.ious[1, 1][0, 0] == 0.5


def test_rle_from_string_round_trip():
    rng = np.random.default_rng(3)
    for _ in range(20):
        m = (rng.random((int(rng.integers(1, 60)), int(rng.integers(1, 60)))) < rng.random()).astype(np.uint8)
        cnts = O.rle_counts(m)
        s = ops.rle_to_string(cnts)
        assert np.array_equal(ops.rle_from_string(s), cnts) and np.array_equal(ops.rle_from_string(s.decode()), cnts)
        h, w, c2 = EV.gt_rle({"size": list(m.shape), "counts": s.decode()})
        assert (h, w) == m.shape and np.array_equal(c2, cnts)
        assert np.array_equal(EV.gt_rle(m)[2], cnts)
        assert np.array_equal(EV.gt_rle({"size": list(m.shape), "counts": cnts.tolist()})[2], cnts)
    with pytest.raises(ValueError, match="polygon"):
        EV.gt_rle([[0, 0, 10, 0, 10, 10]])


def test_host_summarize_matches_oracle():
    rng = np.random.default_rng(5)
    gts, images = [], []
    for im in range(6):
        for j in range(int(rng.integers(0, 6))):
            x, y, w, h = rng.uniform(0, 300, 2).tolist() + rng.uniform(5, 150, 2).tolist()
            gts.append(box_gt(im, int(rng.integers(1, 4)), (x, y, w, h), iscrowd=int(rng.random() < 0.1)))
        n = int(rng.integers(0, 12))
        b = rng.uniform(0, 300, (n, 2)); s = rng.uniform(5, 150, (n, 2))
        images.append(det(im, np.hstack([b, b + s]), rng.random(n), rng.integers(1, 4, n)))
    E = CO.evaluate(gts, images, [1, 2, 3], "bbox")
    assert np.array_equal(EV.summarize_stats(E.eval["precision"], E.eval["recall"]), E.stats)
    pc = EV.per_class_ap(E.eval["precision"])
    for lo, hi in ((0, 9), (0, 0)):
        p = E.eval["precision"][lo:hi + 1, :, :, 0, 2]
        key = "0.50:%.2f" % (0.95 if hi == 9 else 0.5)
        assert pc[key]["mean"] == np.mean(p[p > -1])


@pytest.mark.skipif(not os.path.exists(GOLD_PATH), reason="fixture not generated")
def test_oracle_matches_reference_fixture():
    G = np.load(GOLD_PATH, allow_pickle=False)
    import json
    for iou_type in ("bbox", "segm"):
        data = json.loads(str(G["inputs"]))
        images = [(im["image_id"], np.asarray(im["boxes"], np.float32).reshape(-1, 4), np.asarray(im["scores"], np.float32),
                   np.asarray(im["cls"], np.int64), im.get("segms")) for im in data["images"]]
        results = CO.format_results(images, data["cat_ids"], iou_type)
        ref = json.loads(str(G[iou_type + "/results"]))
        assert len(results) == len(ref)
        for a, b in zip(results, ref):               # the reference's own formatting, bit for bit
            assert a["image_id"] == b["image_id"] and a["category_id"] == b["category_id"] and a["score"] == b["score"]
            if iou_type == "bbox":
                assert a["bbox"] == b["bbox"]
            else:
                assert a["segmentation"] == b["segmentation"]
        E = CO.evaluate(data["gts"], images, data["cat_ids"], iou_type)
        for key in ("precision", "recall", "scores"):
            assert np.array_equal(E.eval[key], G[iou_type + "/" + key])
        assert np.array_equal(E.stats, G[iou_type + "/stats"])
        # log_detection_eval_metrics, executed: the slices it took and the values it logged
        pc = EV.per_class_ap(E.eval["precision"])
        logged = [str(s) for s in G[iou_type + "/logged"]]
        want = []
        for key in ("0.50:0.95", "0.50:0.50"):
            want += ["{:.3f}".format(v) for v in pc[key]["per_class"]] + ["{:.3f}".format(pc[key]["mean"])]
        assert logged == want
        slices = G[iou_type + "/slices"]                # rows: (lo, hi + 1, class K index or -1, area, maxDet)
        K = len(data["cat_ids"])
        want_slices = [(0, hi, k, 0, 2) for hi in (10, 1) for k in [-1] + list(range(K))]
        assert [tuple(int(v) for v in r) for r in slices] == want_slices


def test_against_pycocotools():
    pytest.importorskip("pycocotools")
    from pycocotools.coco import COCO
    from pycocotools.cocoeval import COCOeval
    rng = np.random.default_rng(11)
    H, W = 60, 80
    imgs, anns, images = [], [], []
    for im in range(8):
        imgs.append({"id": im + 1, "height": H, "width": W})
        for j in range(int(rng.integers(0, 5))):
            m = np.zeros((H, W), np.uint8)
            y, x = int(rng.integers(0, H - 5)), int(rng.integers(0, W - 5))
            m[y:y + int(rng.integers(3, 40)), x:x + int(rng.integers(3, 50))] = 1
            rle = O.mask_encode(m)
            ys, xs = np.nonzero(m)
            anns.append({"id": len(anns) + 1, "image_id": im + 1, "category_id": int(rng.integers(1, 4)),
                         "iscrowd": int(rng.random() < 0.15), "area": float(m.sum()),
                         "bbox": [float(xs.min()), float(ys.min()), float(np.ptp(xs) + 1), float(np.ptp(ys) + 1)],
                         "segmentation": {"size": [H, W], "counts": rle["counts"].decode()}})
        n = int(rng.integers(0, 8))
        b = rng.uniform(0, 60, (n, 2)); s = rng.uniform(3, 40, (n, 2))
        segs = []
        for i in range(n):
            m = np.zeros((H, W), np.uint8)
            m[int(b[i, 1]) % H:int(b[i, 1] + s[i, 1]), int(b[i, 0]) % W:int(b[i, 0] + s[i, 0])] = 1
            segs.append({"size": [H, W], "counts": O.mask_encode(m)["counts"].decode()})
        images.append((im + 1, np.hstack([b, b + s]).astype(np.float32), rng.random(n).astype(np.float32),
                       rng.integers(1, 4, n), segs))
    cats = [{"id": c, "name": str(c)} for c in (1, 2, 3)]
    gt = COCO()
    gt.dataset = {"images": imgs, "annotations": anns, "categories": cats}
    gt.createIndex()
    for iou_type in ("bbox", "segm"):
        res = CO.format_results(images, [1, 2, 3], iou_type)
        if not res:
            continue
        E = COCOeval(gt, gt.loadRes(res), iou_type)
        E.evaluate(); E.accumulate(); E.summarize()
        mine = CO.evaluate(anns, images, [1, 2, 3], iou_type)
        for key in ("precision", "recall", "scores"):
            assert np.array_equal(E.eval[key], mine.eval[key])
        assert np.array_equal(E.stats, mine.stats)
