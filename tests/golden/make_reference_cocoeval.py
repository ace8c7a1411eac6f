"""Fixtures for COCO box / mask AP: the reference's OWN result formatting and AP slicing executed in the build container.

Compiled from the reference files by AST, unmodified: `xyxy_to_xywh` (bbox/bbox_transform.py:241-254) and the methods
`bbox_results_one_category`, `segms_results_one_category` and `log_detection_eval_metrics` (dataset/base_dataset.py:626-716),
driven the way evaluate_boxes / evaluate_masks drive them (class-major, image ids sorted, a JSON round trip of the
results).  pycocotools is not in this image and the reference does not vendor it, so the stub COCO / COCOeval they call
is backed by the numpy restatement (tests/coco_oracle.py).  The module-level `np` they see is numpy with the `np.float`
alias (removed from numpy 1.24) restored; `sys` is a namespace whose `stdout` the logging tee may replace.
What the fixture pins to reference-executed code: the float64 box formatting (w = x2 - x1 + 1), the result order and
fields, and which precision slices the per-class AP lines average.  COCOeval itself stays pinned to its published
algorithm.

Run (build container only):  python tests/golden/make_reference_cocoeval.py  ->  tests/golden/reference_cocoeval.npz
"""
import ast
import json
import os
import sys
import tempfile
import types

import numpy

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import coco_oracle as CO  # noqa: E402
from oracle import oracle as O  # noqa: E402

REF = "/root/reference/upsnet"


def _fn(path, name):
    src = open(path).read()
    return [n for n in ast.walk(ast.parse(src)) if isinstance(n, ast.FunctionDef) and n.name == name][0]


class _NumpyWithFloat(types.ModuleType):
    def __getattr__(self, name):
        return float if name == "float" else getattr(numpy, name)


np = _NumpyWithFloat("numpy")


def reference_functions(logger):
    ns = {"np": np}
    exec(compile(ast.Module(body=[_fn(REF + "/bbox/bbox_transform.py", "xyxy_to_xywh")], type_ignores=[]),
                 "bbox_transform.py:241-254", "exec"), ns)
    ns2 = {"np": np, "bbox_transform": types.SimpleNamespace(xyxy_to_xywh=ns["xyxy_to_xywh"]), "logger": logger,
           "sys": types.SimpleNamespace(stdout=sys.stdout)}
    body = [_fn(REF + "/dataset/base_dataset.py", n)
            for n in ("bbox_results_one_category", "segms_results_one_category", "log_detection_eval_metrics")]
    exec(compile(ast.Module(body=body, type_ignores=[]), "base_dataset.py:626-716", "exec"), ns2)
    return ns2


class Logger:
    def __init__(self):
        self.lines = []

    def info(self, msg):
        self.lines.append(msg)


class Recorder:
    """coco_eval.eval['precision'] that records the index of every slice taken."""
    def __init__(self, a):
        self.a, self.keys = a, []

    def __getitem__(self, key):
        lo_hi, _, k, a, m = key
        self.keys.append((lo_hi.start, lo_hi.stop, -1 if isinstance(k, slice) else int(k), int(a), int(m)))
        return self.a[key]


def dataset(rng):
    """6 images at 64x96, categories 1, 3, 7, 9: crowds, all area ranges present, exact score ties, empty images."""
    H, W = 64, 96
    cat_ids = [1, 3, 7, 9]
    gts, images = [], []
    for i, image_id in enumerate([40, 12, 33, 7, 25, 18]):
        for _ in range(0 if i == 4 else int(rng.integers(1, 6))):
            w, h = (int(v) for v in rng.integers(3, 60, 2))
            x, y = int(rng.integers(0, W - w)), int(rng.integers(0, H - h))
            m = numpy.zeros((H, W), numpy.uint8)
            m[y:y + h, x:x + w] = 1
            gts.append({"id": len(gts) + 1, "image_id": image_id, "category_id": cat_ids[int(rng.integers(0, 4))],
                        "iscrowd": int(rng.random() < 0.15), "area": float(w * h), "bbox": [float(x), float(y), float(w), float(h)],
                        "segmentation": {"size": [H, W], "counts": O.mask_encode(m)["counts"].decode()}})
        n = 0 if i == 2 else int(rng.integers(2, 9))
        xy = rng.uniform(0, 80, (n, 2)); wh = rng.uniform(2, 50, (n, 2))
        boxes = numpy.hstack([xy, numpy.minimum(xy + wh, [W - 1, H - 1])]).astype(numpy.float32)
        scores = (numpy.round(rng.uniform(0, 1, n) * 8) / 8).astype(numpy.float32)
        cls = rng.integers(1, 5, n)
        segms = []
        for b in boxes.astype(int):
            m = numpy.zeros((H, W), numpy.uint8)
            m[b[1]:b[3] + 1, b[0]:b[2] + 1] = 1
            segms.append({"size": [H, W], "counts": O.mask_encode(m)["counts"].decode()})
        images.append({"image_id": image_id, "boxes": boxes.tolist(), "scores": scores.tolist(), "cls": cls.tolist(),
                       "segms": segms})
    return {"cat_ids": cat_ids, "gts": gts, "images": images}


def main():
    data = dataset(numpy.random.default_rng(2026))
    out = {"inputs": numpy.array(json.dumps(data))}
    classes = ["__background__"] + ["c%d" % c for c in data["cat_ids"]]
    by_id = sorted(data["images"], key=lambda im: im["image_id"])
    for iou_type in ("bbox", "segm"):
        logger = Logger()
        ref = reference_functions(logger)
        coco = types.SimpleNamespace(getImgIds=lambda: [im["image_id"] for im in data["images"]])
        self = types.SimpleNamespace(dataset=types.SimpleNamespace(COCO=coco, classes=classes))
        results = []
        for j, cat_id in enumerate(data["cat_ids"], start=1):           # evaluate_boxes / evaluate_masks loop
            boxes, segms = [], []
            for im in by_id:                                           # im_post's per-class arrays: [x1 y1 x2 y2 score]
                sel = numpy.flatnonzero(numpy.asarray(im["cls"]) == j)
                b = numpy.asarray(im["boxes"], numpy.float32).reshape(-1, 4)[sel]
                boxes.append(numpy.hstack([b, numpy.asarray(im["scores"], numpy.float32)[sel, None]]))
                segms.append([im["segms"][d] for d in sel])
            if iou_type == "bbox":
                results.extend(ref["bbox_results_one_category"](self, boxes, cat_id))
            else:
                results.extend(ref["segms_results_one_category"](self, boxes, segms, cat_id))
        text = json.dumps(results)                                     # json.dump + COCO.loadRes's json.load
        loaded = json.loads(text)
        E = CO.COCOeval(data["gts"], CO.load_res(loaded, iou_type), [im["image_id"] for im in data["images"]],
                        data["cat_ids"], iou_type)
        E.evaluate()
        E.accumulate()
        rec = Recorder(E.eval["precision"])
        stub = types.SimpleNamespace(params=types.SimpleNamespace(iouThrs=CO.IOU_THRS), eval={"precision": rec},
                                     summarize=E.summarize)
        with tempfile.TemporaryDirectory() as tmp:
            ref["log_detection_eval_metrics"](self, stub, os.path.join(tmp, "detection_results.txt"))
        logged = [s for s in logger.lines if not s.startswith("~")]
        pre = iou_type + "/"
        out[pre + "results"] = numpy.array(text)
        for key in ("precision", "recall", "scores"):
            out[pre + key] = E.eval[key]
        out[pre + "stats"] = E.stats
        out[pre + "logged"] = numpy.array(logged)
        out[pre + "slices"] = numpy.array(rec.keys, numpy.int64)
    numpy.savez_compressed(os.path.join(HERE, "reference_cocoeval.npz"), **out)
    print("wrote reference_cocoeval.npz:", {k: getattr(v, "shape", None) for k, v in out.items()})


if __name__ == "__main__":
    main()
