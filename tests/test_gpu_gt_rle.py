"""Device ground-truth rasteriser (csrc/gt_rle.cu, ops.ann_to_rle, DetectionAP with polygon ground truths) against the
annToRLE restatement (tests/gt_rle_oracle.py): run for run at COCO and Cityscapes sizes, repeatable on any stream, bad
input refused before any launch, and mask AP from polygons bit-identical to mask AP from the oracle's RLEs and to the
COCOeval restatement."""
import functools

import numpy as np
import pytest
import torch

import coco_oracle as CO
import gt_rle_oracle as GO
import test_gpu_cocoeval as TC
from oracle import oracle as O
from proposal_target_oracle import rle_decode

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


def star(rng, cx, cy, r, n):
    a = np.sort(rng.uniform(0, 2 * np.pi, n))
    rr = r * rng.uniform(0.6, 1.0, n)
    return [float(round(v, 2)) for xy in zip(cx + rr * np.cos(a), cy + rr * np.sin(a)) for v in xy]


def crowd_rle(rng, h, w, compressed):
    m = np.zeros((h, w), np.uint8)
    y, x = int(rng.integers(0, h - 1)), int(rng.integers(0, w - 1))
    m[y:y + int(rng.integers(1, h // 3 + 2)), x:x + int(rng.integers(1, w // 3 + 2))] = 1
    m[rng.random((h, w)) < 0.002] ^= 1
    if compressed:
        return {"size": [h, w], "counts": O.mask_encode(m)["counts"].decode()}
    return {"size": [h, w], "counts": GO.encode_flat(m.T.reshape(-1)).tolist()}


def random_segms(rng, h, w, G, huge=0):
    """G COCO-like segmentations: polygon lists of 1-3 parts (stars, border crossers, self-intersecting, full-width
    edges, 5c + .5 boundaries), box lists, crowd RLE dicts (compressed and not), and `huge` stars of thousands of
    vertices."""
    out = []
    for i in range(G):
        r = rng.random()
        if i < huge:
            out.append([star(rng, rng.uniform(0, w), rng.uniform(0, h), rng.uniform(0.2, 0.6) * min(h, w),
                             int(rng.integers(1500, 4000)))])
        elif r < 0.08:
            out.append(crowd_rle(rng, h, w, rng.random() < 0.5))
        elif r < 0.13:
            out.append([[float(v) for v in np.r_[rng.uniform(-5, [w, h]), rng.uniform(0, 300, 2)]]
                        for _ in range(int(rng.integers(1, 3)))])
        else:
            out.append([GO.random_polygon(rng, h, w, int(rng.integers(0, 6))) for _ in range(int(rng.integers(1, 4)))])
    return out


def device_runs(segms, h, w):
    from upsnet_b200 import operators as ops
    err = torch.zeros((1,), dtype=torch.int32, device=DEV)
    counts, offs = ops.ann_to_rle(segms, h, w, DEV, err=err)
    assert int(err.item()) == 0
    return counts.cpu().numpy().view(np.uint32), offs.cpu().numpy()


CASES = [(480, 640, 1, 0), (480, 640, 7, 0), (640, 427, 60, 1), (640, 640, 1024, 2), (1024, 2048, 40, 2),
         (7, 300, 30, 0)]


@pytest.mark.parametrize("h,w,G,huge", CASES, ids=["%dx%d_g%d" % c[:3] for c in CASES])
def test_kernel_matches_oracle_run_for_run(h, w, G, huge):
    rng = np.random.default_rng([h, w, G])
    segms = random_segms(rng, h, w, G, huge)
    c, o = device_runs(segms, h, w)
    assert o.shape == (G + 1,) and o[0] == 0
    for g, s in enumerate(segms):
        want = GO.ann_to_rle(s, h, w)["counts"]
        got = c[o[g]:o[g + 1]]
        assert np.array_equal(got, want), "annotation %d of %d (%s): %d runs vs %d" % (g, G, type(s).__name__, got.size, want.size)


def test_full_width_edges_and_band_borders():
    # rectangles spanning the whole width at 1024 x 2048 (every band of the column-major order), their lower edge on the
    # last row (the y = h spill), one clipped polygon crossing every band border, and one overlapping part per annotation
    h, w = 1024, 2048
    segms = [[[-3, 0.1, w + 4, 0.1, w + 4, h + 7, -3, h + 7]], [[0, 500, w, 500, w, h, 0, h], [10, 10, 40, 900, 70, 10]],
             [[0.5, 0.5, w - 0.5, 3, 5, h - 0.5]], [[1000, 1023.9, 1001, 1023.9, 1001, 1024.1]]]
    c, o = device_runs(segms, h, w)
    for g, s in enumerate(segms):
        assert np.array_equal(c[o[g]:o[g + 1]], GO.ann_to_rle(s, h, w)["counts"]), g


def test_repeatable_and_side_stream():
    from upsnet_b200 import operators as ops
    rng = np.random.default_rng(4)
    segms = random_segms(rng, 480, 640, 300, 1)
    a = [x.cpu().numpy() for x in ops.ann_to_rle(segms, 480, 640, DEV)]
    b = [x.cpu().numpy() for x in ops.ann_to_rle(segms, 480, 640, DEV)]
    s = torch.cuda.Stream(DEV)
    with torch.cuda.stream(s):
        out = ops.ann_to_rle(segms, 480, 640, DEV)
    s.synchronize()
    c = [x.cpu().numpy() for x in out]
    n = int(a[1][-1])
    for x in (b, c):
        assert np.array_equal(a[1], x[1]) and np.array_equal(a[0][:n], x[0][:n])


def test_bad_input_raises_before_any_launch():
    from upsnet_b200 import DetectionAP
    from upsnet_b200 import operators as ops
    ap = DetectionAP([{"id": 1}], "segm")
    g = {"category_id": 1, "iscrowd": 0, "area": 16.0, "bbox": [1.0, 1.0, 4.0, 4.0]}
    empty = (torch.zeros((0, 8), dtype=torch.int32, device=DEV), torch.zeros(0, dtype=torch.int32, device=DEV))
    det = (TC.t(np.zeros((0, 4), np.float32)), TC.t(np.zeros(0, np.float32)), TC.t(np.zeros(0, np.int64)))
    with pytest.raises(ValueError, match="polygon"):                 # no im_size: the image record's size is unknown
        ap.update(1, [dict(g, segmentation=[[0, 0, 4, 0, 4, 4]])], *det, rle=empty)
    with pytest.raises(ValueError, match="empty polygon list"):
        ap.update(1, [dict(g, segmentation=[])], *det, rle=empty, im_size=(20, 30))
    with pytest.raises(ValueError):
        ops.ann_to_rle([[[0, 0, 1]]], 20, 30, DEV)
    torch.cuda.synchronize()
    assert ap._image_ids == [] and int(ap._n_rec.item()) == 0 and int(ap._err.item()) == 0
    assert ap._gt_counts.numel() == 0                                # the rasteriser never ran


@functools.lru_cache(maxsize=None)
def polygon_dataset(seed=21):
    """~60 COCO-like images (480 x 640, a few 640 x 427) with polygon ground truths (crowds as RLE dicts, a few box
    lists), and detections near them whose masks come from ops.im_post_rle."""
    rng = np.random.default_rng(seed)
    sizes = [(480, 640)] * 54 + [(640, 427)] * 6
    ids = rng.permutation(np.arange(3000, 3000 + 3 * len(sizes), 3)).tolist()
    out = []
    for i, ((H, W), image_id) in enumerate(zip(sizes, ids)):
        cls_pool = rng.choice(np.arange(1, 81), 4, replace=False)
        gts, oracle_gts = [], []
        for j in range(0 if i % 17 == 4 else int(rng.integers(1, 10))):
            cx, cy = rng.uniform(0, W), rng.uniform(0, H)
            r = float(np.exp(rng.uniform(np.log(4), np.log(min(H, W) * 0.4))))
            crowd = int(rng.random() < 0.1)
            if crowd:
                seg = crowd_rle(rng, H, W, False)
            elif rng.random() < 0.05:
                seg = [[float(cx), float(cy), float(r), float(r * 0.7)]]
            else:
                seg = [star(rng, cx, cy, r, int(rng.integers(3, 40)))]
                if rng.random() < 0.2:
                    seg.append(star(rng, cx + r, cy, r / 2, int(rng.integers(3, 20))))
            R = GO.ann_to_rle(seg, H, W)
            ys, xs = np.nonzero(rle_decode(np.asarray(R["counts"], np.int64), H, W))
            bbox = [float(xs.min()), float(ys.min()), float(np.ptp(xs) + 1), float(np.ptp(ys) + 1)] if xs.size \
                else [float(cx), float(cy), 1.0, 1.0]
            area = float(CO.rle_area(R)) if rng.random() < 0.8 else float(r * r)
            ann = {"category_id": TC.CAT_IDS[int(rng.choice(cls_pool)) - 1], "iscrowd": crowd, "area": area,
                   "bbox": bbox}
            gts.append(dict(ann, segmentation=seg))
            oracle_gts.append(dict(ann, segmentation={"size": [H, W], "counts": [int(v) for v in R["counts"]]}))
        boxes, cls = [], []
        for g in gts:
            for _ in range(int(rng.integers(0, 3))):
                x, y, w, h = g["bbox"]
                jt = rng.normal(0, 0.08 * max(w, h), 4)
                boxes.append([x + jt[0], y + jt[1], x + w + jt[2], y + h + jt[3]])
                cls.append(TC.CAT_IDS.index(g["category_id"]) + 1 if rng.random() < 0.9 else int(rng.integers(1, 81)))
        for _ in range(int(rng.integers(0, 8))):
            c = rng.uniform([0, 0], [W, H]); s = rng.uniform(4, 300, 2)
            boxes.append([c[0] - s[0] / 2, c[1] - s[1] / 2, c[0] + s[0] / 2, c[1] + s[1] / 2])
            cls.append(int(rng.choice(cls_pool)))
        n = len(boxes)
        b = np.asarray(boxes, np.float32).reshape(-1, 4)
        b[:, 0::2] = np.clip(b[:, 0::2], 0, W - 1); b[:, 1::2] = np.clip(b[:, 1::2], 0, H - 1)
        scores = (np.round(rng.uniform(0.05, 1.0, n) * 20) / 20).astype(np.float32)
        out.append(dict(image_id=image_id, H=H, W=W, gts=gts, oracle_gts=oracle_gts, boxes=b, scores=scores,
                        cls=np.asarray(cls, np.int64), masks=TC.blob_masks(rng, n)))
    return out


def run_ap(data, key):
    from upsnet_b200 import DetectionAP
    from upsnet_b200 import operators as ops
    ap = DetectionAP(TC.CATS, "segm")
    for im in data:
        if len(im["boxes"]):
            cn, rl, ovf = ops.im_post_rle(TC.t(im["boxes"]), TC.t(im["masks"]), TC.t(im["cls"]), im["H"], im["W"])
            assert int(ovf.item()) == 0
        else:
            cn, rl = torch.zeros((0, 16), dtype=torch.int32, device=DEV), torch.zeros(0, dtype=torch.int32, device=DEV)
        ap.update(im["image_id"], im[key], TC.t(im["boxes"]), TC.t(im["scores"]), TC.t(im["cls"]), rle=(cn, rl),
                  im_size=(im["H"], im["W"]))
    return ap.summarize()


def test_end_to_end_polygons_equal_rles_and_oracle():
    data = polygon_dataset()
    assert sum(isinstance(g["segmentation"], list) for im in data for g in im["gts"]) > 200
    res_p = run_ap(data, "gts")
    res_r = run_ap(data, "oracle_gts")
    for key in ("precision", "recall", "scores", "stats"):
        assert np.array_equal(res_p[key], res_r[key]), key
    gts = [dict(g, image_id=im["image_id"]) for im in data for g in im["oracle_gts"]]
    images = [(im["image_id"], im["boxes"], im["scores"], im["cls"],
               [O.mask_encode(m) for m in O.im_post_masks(im["boxes"], im["masks"], im["cls"], im["H"], im["W"])])
              for im in data]
    E = CO.evaluate(gts, images, TC.CAT_IDS, "segm")
    TC.assert_same(res_p, E)
    assert (E.eval["precision"] > 0).any()
