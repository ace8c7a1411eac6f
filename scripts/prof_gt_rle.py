"""Polygon ground truths in DetectionAP('segm'): host time of update() per image with polygon ground truths against the
same set pre-rasterised as RLE dicts, and the rasteriser's kernel time (upsnet_gt_rle: three launches) from CUDA events.

The set is COCO-val-like: 480 x 640 and 640 x 427 images, about 7 instances per image (1 to 20), 1-3 polygons each with
a realistic vertex-count spread (log-uniform 4 to 400), one crowd RLE in ten.  Detections are empty, so update() time is
the ground-truth work plus the matching launch.  Prints one JSON line; the card name and power limit are read in the same
run.  python scripts/prof_gt_rle.py [--images 500] [--reps 20]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def dataset(n, seed=0):
    import gt_rle_oracle as GO
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        H, W = ((480, 640), (640, 427))[i % 3 == 2]
        segms = []
        for _ in range(int(np.clip(rng.poisson(7), 1, 20))):
            if rng.random() < 0.1:
                m = np.zeros((H, W), np.uint8)
                y, x = int(rng.integers(0, H - 40)), int(rng.integers(0, W - 40))
                m[y:y + int(rng.integers(10, 120)), x:x + int(rng.integers(10, 120))] = 1
                segms.append({"size": [H, W], "counts": GO.encode_flat(m.T.reshape(-1)).tolist()})
                continue
            cx, cy = rng.uniform(0, W), rng.uniform(0, H)
            r = float(np.exp(rng.uniform(np.log(5), np.log(200))))
            parts = []
            for j in range(int(rng.choice([1, 1, 1, 2, 3]))):
                k = int(np.exp(rng.uniform(np.log(4), np.log(400))))
                a = np.sort(rng.uniform(0, 2 * np.pi, k))
                rr = r / (1 + j) * rng.uniform(0.6, 1.0, k)
                ox = (cx + rr * np.cos(a) + j * r).clip(0, W - 1)
                oy = (cy + rr * np.sin(a)).clip(0, H - 1)
                parts.append([round(float(v), 2) for v in np.stack([ox, oy], 1).reshape(-1)])
            segms.append(parts)
        out.append((H, W, segms))
    return out


def main():
    ap_ = argparse.ArgumentParser()
    ap_.add_argument("--images", type=int, default=500)
    ap_.add_argument("--reps", type=int, default=20)
    args = ap_.parse_args()
    import gt_rle_oracle as GO
    from upsnet_b200 import DetectionAP
    from upsnet_b200 import operators as ops
    from upsnet_b200._lib import query_bytes
    dev = torch.device("cuda", 0)
    data = dataset(args.images)
    rles = [[GO.ann_to_rle(s, H, W) for s in segms] for H, W, segms in data]
    rles = [[{"size": r["size"], "counts": [int(v) for v in r["counts"]]} for r in im] for im in rles]
    cats = [{"id": 1}]
    empty = (torch.zeros((0, 16), dtype=torch.int32, device=dev), torch.zeros(0, dtype=torch.int32, device=dev))
    det = (torch.zeros((0, 4), device=dev), torch.zeros(0, device=dev), torch.zeros(0, dtype=torch.int64, device=dev))

    def anns(segms):
        return [{"category_id": 1, "iscrowd": int(isinstance(s, dict)), "area": 100.0, "bbox": [0.0, 0.0, 1.0, 1.0],
                 "segmentation": s} for s in segms]
    sets = {"polygons": [anns(s) for _, _, s in data], "rle_dicts": [anns(r) for r in rles]}

    def run(name):
        ap = DetectionAP(cats, "segm")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i, (H, W, _) in enumerate(data):
            ap.update(i, sets[name][i], *det, rle=empty, im_size=(H, W))
        t1 = time.perf_counter()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        ap.check_errors()
        return (t1 - t0) / len(data) * 1e3, (t2 - t0) / len(data) * 1e3

    for name in sets:                 # warm-up: module load, pinned ring, workspaces
        run(name)
    host = {k: [] for k in sets}
    wall = {k: [] for k in sets}
    for _ in range(3):
        for name in sets:
            h_, w_ = run(name)
            host[name].append(h_)
            wall[name].append(w_)
    # kernel time of the rasteriser alone, per image, from events around upsnet_gt_rle (inputs staged once)
    staged = []
    for H, W, segms in data[:50]:
        pk = ops.pack_segmentations(segms, H, W)
        arrays = ops.gt_rle_arrays(pk)
        buf = [torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).copy()).to(dev) for a in arrays]
        G = len(pk.ann_poly) - 1
        out = (torch.empty((max(pk.bound, 1),), dtype=torch.int32, device=dev), torch.empty((G + 1,), dtype=torch.int64, device=dev))
        ws = torch.empty((max(1, query_bytes("gt_rle_workspace_bytes", G, H, W)),), dtype=torch.uint8, device=dev)
        staged.append((pk, H, W, buf, out, ws))
    err = torch.zeros((1,), dtype=torch.int32, device=dev)

    def launch_all():
        for pk, H, W, buf, out, ws in staged:
            ops.gt_rle_call(pk, H, W, [C.c_void_p(b.data_ptr()) for b in buf], out[0], out[1], err, ws)
    launch_all()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.reps):
        launch_all()
    e1.record()
    torch.cuda.synchronize()
    kern_ms = e0.elapsed_time(e1) / (args.reps * len(staged))
    assert int(err.item()) == 0
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    n_ann = sum(len(s) for _, _, s in data)
    n_vert = sum(len(p) // 2 for _, _, s in data for x in s if isinstance(x, list) for p in x)
    print(json.dumps({
        "gpu": smi[0] if smi else "unknown", "images": len(data), "annotations_per_image": n_ann / len(data),
        "vertices_per_image": n_vert / len(data),
        "update_host_ms_per_image": {k: min(v) for k, v in host.items()},
        "update_wall_ms_per_image": {k: min(v) for k, v in wall.items()},
        "gt_rle_kernel_ms_per_image": kern_ms}))


if __name__ == "__main__":
    main()
