"""Generates tests/golden/reference_combined.npz by EXECUTING the reference's combined panoptic result (build container
only: the reference tree is not present on the GPU box).  Run: python tests/golden/make_reference_combined.py

Executed, unmodified, from /root/reference/upsnet/dataset/base_dataset.py, extracted by AST as make_reference_pq.py does
(the module itself pulls pycocotools / Cython at import):
  :373-403  BaseDataset.get_combined_pan_result   (per-class lists concatenated, argsort by score, Pool over images)
  :405-449  BaseDataset._merge_pred_single_core   (skip rules, claims, stuff area limit, merge)
Stubs:
  * config.dataset.num_seg_classes / num_classes, set per case;
  * multiprocessing: cpu_count() = 1 and a synchronous Pool, so every case is one image per call (np.array_split over
    ragged per-image lists raises under numpy 2 for two or more images with different detection counts);
  * pycocotools.mask.decode: pycocotools is not installed and the reference does not vendor it, so it is the repository's
    restated decoder (oracle.rle_from_string + rle_decode).  Codec parity stays unpinned, as in the other fixtures.

Detections are stored in engine order (classes mixed); the per-class lists handed to the reference keep that order within
a class, as im_post builds them.  For each case the file records whether the executed argsort gave the order of rule 2
(order_ok): exact-score ties have no order the reference guarantees.  The seeded 1024x2048 case is rebuilt by the tests
from tests/combined_oracle.large_case(), so only the sha256 of the reference's output is stored.
"""
import ast
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import combined_oracle as CO  # noqa: E402
from oracle import oracle as O  # noqa: E402

REF = "/root/reference/upsnet"


class _Result:
    def __init__(self, v):
        self.v = v

    def get(self):
        return self.v


class _Pool:
    def __init__(self, processes=None):
        pass

    def apply_async(self, f, args):
        return _Result(f(*args))

    def close(self):
        pass

    def join(self):
        pass


def _decode(rle):
    return O.rle_decode(O.rle_from_string(rle["counts"]), int(rle["size"][0]), int(rle["size"][1]))


def load_reference():
    pc = types.ModuleType("pycocotools")
    pm = types.ModuleType("pycocotools.mask")
    pm.decode = _decode
    pc.mask = pm
    sys.modules["pycocotools"], sys.modules["pycocotools.mask"] = pc, pm
    path = os.path.join(REF, "dataset", "base_dataset.py")
    tree = ast.parse(open(path).read())
    want = ("get_combined_pan_result", "_merge_pred_single_core")
    nodes = [n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name in want]
    for n in nodes:
        n.decorator_list = []                             # @staticmethod is re-applied below
    mp = types.SimpleNamespace(cpu_count=lambda: 1, Pool=_Pool)
    config = types.SimpleNamespace(dataset=types.SimpleNamespace(num_seg_classes=19, num_classes=9))
    ns = {"np": np, "multiprocessing": mp, "config": config, "__file__": path}
    exec(compile(ast.Module(body=nodes, type_ignores=[]), "base_dataset.py:373-449", "exec"), ns)
    ns["BaseDataset"] = type("BaseDataset", (), {"get_combined_pan_result": ns["get_combined_pan_result"],
                                                 "_merge_pred_single_core": staticmethod(ns["_merge_pred_single_core"])})
    return ns


def reference_inputs(sem, scores, cls, runs, num_classes):
    """The test script's all_ssegs / all_boxes / all_masks for one image (boxes are irrelevant to the merge: zeros)."""
    H, W = sem.shape
    boxes = [[np.zeros((0, 5), np.float32)]] + [[None] for _ in range(1, num_classes)]
    masks = [[[]]] + [[None] for _ in range(1, num_classes)]
    for j in range(1, num_classes):
        sel = np.flatnonzero(cls == j)
        b = np.zeros((sel.size, 5), np.float32)
        b[:, 4] = scores[sel]
        boxes[j][0] = b
        masks[j][0] = [{"size": [H, W], "counts": O.rle_to_string(runs[d]).decode()} for d in sel]
    return [sem.copy()], boxes, masks


def run_reference(ns, case):
    sem, scores, cls, runs, (nsc, nc, st, ft, lim) = case
    ns["config"].dataset.num_seg_classes, ns["config"].dataset.num_classes = nsc, nc
    segs, boxes, masks = reference_inputs(sem, scores, cls, runs, nc)
    ds = ns["BaseDataset"]()
    pans = ds.get_combined_pan_result(segs, boxes, masks, score_threshold=st, fraction_threshold=ft, stuff_area_limit=lim)
    assert len(pans) == 1
    # the order the executed argsort gave vs rule 2 (stable argsort reversed over the class-ascending concatenation)
    sc_cat = np.concatenate([boxes[j][0][:, 4] for j in range(1, nc)])
    order_ok = bool(np.array_equal(np.argsort(sc_cat)[::-1], np.argsort(sc_cat, kind="stable")[::-1]))
    return pans[0], order_ok


def rect(H, W, y0, y1, x0, x1):
    m = np.zeros((H, W), np.uint8)
    m[y0:y1, x0:x1] = 1
    return m


def small_cases(rng):
    H, W = 40, 56
    cs = (19, 9, 0.6, 0.7, 64)                            # Cityscapes class counts, a small stuff limit
    cases = {}
    sem = CO.semantic_map(rng, H, W, 19, block=8)

    def case(masks, scores, cls, params=cs, s=sem):
        return (s, np.asarray(scores, np.float32), np.asarray(cls, np.int64), [O.rle_counts(m) for m in masks], params)

    # distinct scores across classes, overlapping masks: the later ones lose their claimed pixels
    ms = [rect(H, W, 2, 20, 2, 20), rect(H, W, 10, 30, 10, 30), rect(H, W, 5, 35, 30, 50), rect(H, W, 0, 8, 0, 56)]
    cases["order_across_classes"] = case(ms, [0.9, 0.8, 0.95, 0.7], [3, 1, 8, 5])
    f6 = np.float32(0.6)
    cases["score_at_threshold"] = case(ms[:2], [f6, np.nextafter(f6, np.float32(0))], [2, 4])
    # fraction exactly 7/10 (kept under numpy 2) and 69/100 (dropped)
    a = rect(H, W, 0, 3, 0, 1)                                             # 3 pixels of column 0
    b = rect(H, W, 0, 10, 0, 1)                                            # 10 pixels: 7 free
    cases["fraction_7_of_10"] = case([a, b], [0.9, 0.8], [1, 2])
    a = rect(H, W, 0, 20, 0, 1) | rect(H, W, 0, 11, 1, 2)                  # 31 pixels
    b = rect(H, W, 0, 20, 0, 5)                                            # 100 pixels: 69 free
    cases["fraction_69_of_100"] = case([a, b], [0.9, 0.8], [1, 2])
    cases["empty_mask"] = case([np.zeros((H, W), np.uint8), rect(H, W, 4, 9, 4, 9)], [0.99, 0.7], [3, 3])
    cases["covered_mask"] = case([rect(H, W, 0, 20, 0, 20), rect(H, W, 5, 10, 5, 10)], [0.9, 0.8], [1, 1])
    cases["none_above_threshold"] = case(ms, [0.5, 0.1, 0.59, 0.0], [1, 2, 3, 4])
    cases["no_detections"] = case([], [], [])
    # stuff area exactly at the limit and one below: class 0 with 64 pixels, class 1 with 63
    s2 = np.full((H, W), 5, np.uint8)
    s2[0:8, 0:8] = 0
    s2[10:17, 10:19] = 1
    cases["stuff_limit"] = case([rect(H, W, 30, 35, 30, 35)], [0.9], [2], s=s2)
    # thing-class semantic pixels without an instance -> 255; 255 void stays 255
    s3 = np.full((H, W), 3, np.uint8)
    s3[:, 20:40] = 14
    s3[0:5, :] = 255
    cases["thing_without_instance"] = case([rect(H, W, 0, 40, 25, 30)], [0.8], [4], params=(19, 9, 0.6, 0.7, 16), s=s3)
    cases["large_instance"] = case([rect(H, W, 3, 38, 2, 30)], [0.9], [6])
    # several instances of one class, and of two classes interleaved by score
    ms5 = [rect(H, W, 0, 10, 10 * k, 10 * k + 8) for k in range(5)] + [rect(H, W, 20, 30, 10 * k, 10 * k + 8) for k in range(5)]
    cases["several_instances"] = case(ms5, [0.9 - 0.02 * k for k in range(10)], [7] * 5 + [7, 2, 7, 2, 7])
    # full-height masks: the runs of ones cross column boundaries
    cases["full_height"] = case([rect(H, W, 0, H, 5, 17), rect(H, W, 0, H, 12, 30), rect(H, W, 0, 20, 29, 40)],
                                [0.9, 0.85, 0.8], [1, 5, 8])
    # >= 256 kept instances of one class: the 256th writes 0 and leaves its pixels free for a later detection
    Hb, Wb = 48, 64
    sb = CO.semantic_map(rng, Hb, Wb, 19, block=8)
    cells = [rect(Hb, Wb, 2 * (k % 24), 2 * (k % 24) + 2, 2 * (k // 24), 2 * (k // 24) + 2) for k in range(300)]
    sc = (0.99 - 0.0001 * np.arange(300)).astype(np.float32)
    over = rect(Hb, Wb, 2 * (255 % 24), 2 * (255 % 24) + 2, 2 * (255 // 24), 2 * (255 // 24) + 2)   # the 256th's cell
    cases["wrap_256"] = (sb, np.concatenate([sc, [0.6]]).astype(np.float32), np.array([3] * 300 + [4], np.int64),
                         [O.rle_counts(m) for m in cells + [over]], cs)
    # COCO class counts (133 / 81): classes up to 80, id_last_stuff = 52
    s4 = CO.semantic_map(rng, H, W, 133, block=4)
    sc4, cl4, rn4 = CO.random_detections(rng, H, W, 30, 81)
    cases["coco_random"] = (s4, sc4, cl4, rn4, (133, 81, 0.6, 0.7, 16))
    sc5, cl5, rn5 = CO.random_detections(rng, H, W, 40, 9)
    cases["cityscapes_random"] = (sem, sc5, cl5, rn5, cs)
    # the defaults (score 0.6, fraction 0.7, stuff limit 4096) on a 64x96 image: every stuff class is under the limit
    sc6, cl6, rn6 = CO.random_detections(rng, 64, 96, 25, 9)
    cases["defaults"] = (CO.semantic_map(rng, 64, 96, 19, block=8), sc6, cl6, rn6, (19, 9, 0.6, 0.7, 4096))
    # exact score ties within one class and across classes
    ms7 = [rect(H, W, 0, 20, 0, 20), rect(H, W, 5, 25, 5, 25), rect(H, W, 10, 30, 10, 30), rect(H, W, 15, 35, 15, 35),
           rect(H, W, 0, 40, 12, 22), rect(H, W, 20, 40, 0, 40)]
    cases["ties_within_class"] = case(ms7, [0.8] * 6, [2] * 6, params=(19, 9, 0.6, 0.5, 64))
    cases["ties_across_classes"] = case(ms7, [0.8, 0.7, 0.8, 0.8, 0.7, 0.8], [5, 2, 1, 5, 2, 8], params=(19, 9, 0.6, 0.5, 64))
    sc8 = np.round(rng.uniform(0.6, 1.0, 40), 1).astype(np.float32)                             # many ties
    _, cl8, rn8 = CO.random_detections(rng, H, W, 40, 9)
    cases["ties_random"] = (sem, sc8, cl8, rn8, (19, 9, 0.6, 0.5, 64))
    return cases


def main():
    ns = load_reference()
    rng = np.random.default_rng(373)
    cases = small_cases(rng)
    out = {}
    names = sorted(cases)
    for name in names:
        sem, scores, cls, runs, params = cases[name]
        pan, order_ok = run_reference(ns, cases[name])
        out[name + "/sem"] = sem
        out[name + "/scores"] = scores
        out[name + "/cls"] = cls
        out[name + "/runs"] = np.concatenate([np.asarray(r, np.uint32) for r in runs] + [np.zeros(0, np.uint32)])
        out[name + "/run_off"] = np.cumsum([0] + [len(r) for r in runs]).astype(np.int64)
        out[name + "/params"] = np.array(params, np.float64)
        out[name + "/pan"] = pan
        out[name + "/order_ok"] = np.int64(order_ok)
        same = np.array_equal(pan, CO.combined_pan_result(sem, scores, cls, runs, *params))
        print("%-24s n %3d  instances %3d  order_ok %d  oracle %s" % (name, len(runs), len(np.unique(pan[..., 1])) - 1,
                                                                       order_ok, "==" if same else "!="))
    out["cases"] = np.array(names)
    sem, scores, cls, runs = CO.large_case()
    L = CO.LARGE
    params = (L["num_seg_classes"], L["num_classes"], 0.6, 0.7, 4096)
    pan, order_ok = run_reference(ns, (sem, scores, cls, runs, params))
    out["large/params"] = np.array(params, np.float64)
    out["large/sha256"] = np.array(CO.digest(pan))
    out["large/order_ok"] = np.int64(order_ok)
    out["large/instances"] = np.int64(int((pan[..., 1] > 0).sum()))
    print("%-24s n %3d  instance pixels %d  order_ok %d" % ("large", len(runs), int(out["large/instances"]), order_ok))
    np.savez_compressed(os.path.join(HERE, "reference_combined.npz"), **out)


if __name__ == "__main__":
    main()
