"""Device COCO AP (DetectionAP: upsnet_cocoeval_image / upsnet_cocoeval_accumulate) at the COCO size 800x1333 with 100
detections per image and COCO-like ground truths (7 per image over 3 categories, one crowd): python
scripts/prof_cocoeval.py [images]

Reports, for 'bbox' and 'segm':
  * update() per image: wall time per call over many calls ending in a device synchronise (the host side -- parsing the
    ground-truth RLE strings, staging, the launch -- included), and the device time of the stream between CUDA events;
  * accumulate() over the records of `images` updates (5000 by default, as for COCO val): wall time per call, the copy
    of precision / recall / scores back included;
  * the numpy oracle (tests/coco_oracle.py) on the host: evaluate + accumulate of one image, and of 50 images;
and the card and its power limit."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import upsnet_b200 as U  # noqa: E402
from upsnet_b200 import operators as ops  # noqa: E402
import coco_oracle as CO  # noqa: E402
from oracle import oracle as O  # noqa: E402

H, W, N_DET = 800, 1333, 100
CATS = [{"id": c} for c in range(1, 81)]


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        out = "nvidia-smi unavailable (%s)" % e
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q + ": " + out}


def image(rng):
    cats = rng.choice(np.arange(1, 81), 3, replace=False)
    gts = []
    for j in range(7):
        w, h = (float(v) for v in rng.uniform(20, 400, 2))
        x, y = float(rng.uniform(0, W - w)), float(rng.uniform(0, H - h))
        m = np.zeros((H, W), np.uint8)
        m[int(y):int(y + h), int(x):int(x + w)] = 1
        gts.append({"category_id": int(cats[j % 3]), "iscrowd": int(j == 6), "area": float(m.sum()), "bbox": [x, y, w, h],
                    "segmentation": {"size": [H, W], "counts": O.mask_encode(m)["counts"].decode()}})
    c = rng.uniform([0, 0], [W, H], (N_DET, 2)); s = rng.uniform(10, 400, (N_DET, 2))
    boxes = np.concatenate([c - s / 2, c + s / 2], 1).astype(np.float32)
    boxes[:, 0::2] = np.clip(boxes[:, 0::2], 0, W - 1); boxes[:, 1::2] = np.clip(boxes[:, 1::2], 0, H - 1)
    scores = rng.uniform(0.05, 1, N_DET).astype(np.float32)
    cls = rng.choice(cats, N_DET).astype(np.int64)
    yy, xx = np.mgrid[0:28, 0:28].astype(np.float32)
    masks = np.stack([1.0 / (1.0 + np.exp(((xx - 14) ** 2 + (yy - 14) ** 2 - r * r) / 18.0))
                      for r in rng.uniform(6, 14, N_DET)])[:, None].astype(np.float32)
    return gts, boxes, scores, cls, masks


def measure(iou_type, images, data, dev):
    gts, boxes, scores, cls, masks = data
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)         # noqa: E731
    b, s, c = t(boxes), t(scores), t(cls)
    rle = ops.im_post_rle(b, t(masks), c, H, W)[:2] if iou_type == "segm" else None
    ap = U.DetectionAP(CATS, iou_type)
    for i in range(20):
        ap.update(i, gts, b, s, c, rle=rle, im_size=(H, W))
    ap.accumulate()
    ap.reset()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = min(images, 1000)
    t0 = time.perf_counter()
    ev0.record()
    for i in range(n):
        ap.update(i, gts, b, s, c, rle=rle, im_size=(H, W))
    ev1.record()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) / n * 1e3
    dev_ms = ev0.elapsed_time(ev1) / n
    for i in range(n, images):
        ap.update(i, gts, b, s, c, rle=rle, im_size=(H, W))
    torch.cuda.synchronize()
    acc = []
    for _ in range(5):
        t0 = time.perf_counter()
        ap.accumulate()
        acc.append((time.perf_counter() - t0) * 1e3)
    # the timed path computes the oracle's result (one image)
    ap.reset()
    ap.update(0, gts, b, s, c, rle=rle, im_size=(H, W))
    segms = None
    if iou_type == "segm":
        segms = [O.mask_encode(m) for m in O.im_post_masks(boxes, masks, cls, H, W)]
    one = [(0, boxes, scores, cls, segms)]
    t0 = time.perf_counter()
    E = CO.evaluate([dict(g, image_id=0) for g in gts], one, list(range(1, 81)), iou_type)
    oracle_one = (time.perf_counter() - t0) * 1e3
    assert np.array_equal(ap.accumulate()["precision"], E.eval["precision"])
    many = [(i, boxes, scores, cls, segms) for i in range(50)]
    t0 = time.perf_counter()
    CO.evaluate([dict(g, image_id=i) for i in range(50) for g in gts], many, list(range(1, 81)), iou_type)
    oracle_50 = (time.perf_counter() - t0) * 1e3
    return {"update_wall_ms_per_image": round(wall, 4), "update_device_ms_per_image": round(dev_ms, 4),
            "accumulate_wall_ms_%d_images" % images: [round(v, 2) for v in acc],
            "oracle_host_ms_one_image": round(oracle_one, 1), "oracle_host_ms_50_images": round(oracle_50, 1)}


def main():
    images = int(sys.argv[1]) if len(sys.argv) > 1 else 5000
    dev = torch.device("cuda", 0)
    data = image(np.random.default_rng(0))
    rep = {"card": card(), "size": [H, W], "detections_per_image": N_DET, "gt_per_image": 7}
    for iou_type in ("bbox", "segm"):
        rep[iou_type] = measure(iou_type, images, data, dev)
    print(json.dumps(rep, indent=1))


if __name__ == "__main__":
    main()
