"""Generates tests/golden/reference_pq.npz by EXECUTING the reference's own evaluation code (build container only:
the reference tree is not present on the GPU box).  Run: python tests/golden/make_reference_pq.py

Executed, unmodified, from /root/reference/upsnet/dataset/base_dataset.py, extracted by AST like
make_reference_modules.py does for get_unified_pan_result (the module itself pulls pycocotools / Cython at import):
  :46-97    PQStatCat, PQStat (pq_average)
  :462-511  BaseDataset._converter_2ch_single_core   (2-channel map -> segments_info + RGB id image)
  :513-608  BaseDataset._pq_compute_single_core      (confusion counts, matching, FN / crowd / FP)
and upsnet_end2end_test.py:259-266's restore step with the real cv2.resize(INTER_NEAREST) and the reference's float32
im_info (fx = 1 / im_info[2] is a float32 handed to cv2 as a double).  The restore inputs are rebuilt by the tests from
tests/pq_oracle.py:restore_label, so only cv2's output digest (sha256) is stored.  The 1024x2048 case puts its void
and stray instance numbers in 8x8 blocks, which keeps the fixture about 200 KB.

panopticapi (lib/dataset_devkit) is a git submodule that is absent from the reference tree, so `panopticapi.utils` is
stubbed: rgb2id is the published formula, and IdGenerator restates the published rule (stuff -> the category colour,
things -> the category colour if free, else a fresh random colour near it).  Parity of the colour VALUES is therefore
unpinned; the statistics depend only on which pixels share a colour, which the rule fixes.
"""
import ast
import os
import sys
import types
from collections import defaultdict

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import pq_oracle as P  # noqa: E402  (restore_label, digest: shared with the tests)
REF = "/root/reference/upsnet"

# categories: stuff 0..10, things 11..18 (the unified map's class ids for Cityscapes); distinct colours, none black
CATS = {c: {'id': c, 'isthing': int(c >= 11), 'color': [(37 * c + 20) % 256, (91 * c + 50) % 256, (53 * c + 90) % 256],
            'name': 'c%d' % c} for c in range(19)}


def rgb2id(color):
    if isinstance(color, np.ndarray) and len(color.shape) == 3:
        if color.dtype == np.uint8:
            color = color.astype(np.int32)
        return color[:, :, 0] + 256 * color[:, :, 1] + 256 * 256 * color[:, :, 2]
    return int(color[0] + 256 * color[1] + 256 * 256 * color[2])


class IdGenerator:
    def __init__(self, categories):
        self.taken_colors = {(0, 0, 0)}
        self.categories = categories
        for category in self.categories.values():
            if category['isthing'] == 0:
                self.taken_colors.add(tuple(category['color']))
        self.rng = np.random.RandomState(0)

    def get_color(self, cat_id):
        category = self.categories[cat_id]
        if category['isthing'] == 0:
            return category['color']
        base = tuple(category['color'])
        if base not in self.taken_colors:
            self.taken_colors.add(base)
            return base
        while True:
            color = tuple(int(v) for v in np.clip(np.array(base) + self.rng.randint(-30, 31, size=3), 0, 255))
            if color not in self.taken_colors:
                self.taken_colors.add(color)
                return color


def load_reference():
    pa = types.ModuleType("panopticapi")
    pu = types.ModuleType("panopticapi.utils")
    pu.rgb2id, pu.IdGenerator = rgb2id, IdGenerator
    pa.utils = pu
    sys.modules["panopticapi"], sys.modules["panopticapi.utils"] = pa, pu
    path = os.path.join(REF, "dataset", "base_dataset.py")
    tree = ast.parse(open(path).read())
    want_cls = ("PQStatCat", "PQStat")
    want_fn = ("_converter_2ch_single_core", "_pq_compute_single_core")
    nodes = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name in want_cls]
    nodes += [n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name in want_fn]
    ns = {"np": np, "os": os, "sys": sys, "defaultdict": defaultdict, "vis_panoptic": False, "__file__": path}
    exec(compile(ast.Module(body=nodes, type_ignores=[]), "base_dataset.py:46-97,462-608", "exec"), ns)
    return ns


def run_reference(ns, images, categories):
    """images: list of (pan_2ch uint8 [H,W,3], gt_rgb uint8 [H,W,3], segments_info).  -> (stat [256,4], summary)."""
    idgen = IdGenerator(categories)
    anns, pans = ns["_converter_2ch_single_core"](0, [im[0] for im in images], idgen)
    gt_jsons = [{"segments_info": im[2], "image_id": k} for k, im in enumerate(images)]
    pq_stat = ns["_pq_compute_single_core"](0, gt_jsons, anns, [im[1] for im in images], pans,
                                            [{"id": k} for k in range(len(images))], categories)
    stat = np.zeros((256, 4), np.float64)
    for c, s in pq_stat.pq_per_cat.items():
        stat[c] = (s.iou, s.tp, s.fp, s.fn)
    summary = np.full((3, 4), np.nan)
    per_class = np.full((256, 3), np.nan)
    raises = 0
    try:
        for r, (name, isthing) in enumerate((("All", None), ("Things", True), ("Stuff", False))):
            res, pc = pq_stat.pq_average(categories, isthing=isthing)
            summary[r] = (res['pq'], res['sq'], res['rq'], res['n'])
            if name == "All":
                for c, v in pc.items():
                    per_class[c] = (v['pq'], v['sq'], v['rq'])
    except ZeroDivisionError:
        raises = 1
    return stat, summary, per_class, raises


def gt_image(idmap):
    return np.stack([idmap % 256, (idmap // 256) % 256, idmap // 65536], -1).astype(np.uint8)


def seg(i, cat, area, crowd=0):
    return {"id": int(i), "category_id": int(cat), "iscrowd": int(crowd), "area": int(area), "bbox": [0, 0, 1, 1]}


def table_of(idmap, cats, crowd=()):
    """segments_info with the true pixel areas for every id of `cats` {id: category}."""
    return [seg(i, c, int((idmap == i).sum()), int(i in crowd)) for i, c in cats.items()]


def pan_image(cls, inst):
    return np.stack([cls, inst, np.zeros_like(cls)], -1).astype(np.uint8)


def small_cases(rng):
    H, W = 32, 48
    cases = {}
    # perfect match: two things, one stuff
    gid = np.zeros((H, W), np.int64); gid[:, :] = 1000; gid[4:14, 4:20] = 2000; gid[16:30, 24:44] = 2001
    cls = np.full((H, W), 3); ins = np.zeros((H, W), np.int64)
    cls[4:14, 4:20] = 12; ins[4:14, 4:20] = 1; cls[16:30, 24:44] = 14; ins[16:30, 24:44] = 2
    cases["perfect"] = [(pan_image(cls, ins), gt_image(gid), table_of(gid, {1000: 3, 2000: 12, 2001: 14}))]
    # IoU around 0.5: gt 10x10 = 100 px, prediction 10 x k from column 4: I = 80, union = 20 + 10k
    for name, k in (("iou_above", 13), ("iou_half", 14), ("iou_below", 15)):     # 80/150, 80/160 = 0.5 (no match), 80/170
        gid = np.full((H, W), 8, np.int64); gid[2:12, 2:12] = 7         # background: a stuff segment, not VOID
        cls = np.full((H, W), 255); ins = np.zeros((H, W), np.int64)
        cls[2:12, 4:4 + k] = 11; ins[2:12, 4:4 + k] = 5
        cases[name] = [(pan_image(cls, ins), gt_image(gid), [seg(7, 11, 100), seg(8, 0, H * W - 100)])]
    # category mismatch
    gid = np.zeros((H, W), np.int64); gid[2:20, 2:30] = 9
    cls = np.full((H, W), 255); cls[2:20, 2:30] = 12; ins = np.zeros((H, W), np.int64); ins[2:20, 2:30] = 1
    cases["cat_mismatch"] = [(pan_image(cls, ins), gt_image(gid), [seg(9, 13, 18 * 28)])]
    # VOID gt pixels inside a predicted segment change the union
    gid = np.zeros((H, W), np.int64); gid[0:16, 0:20] = 5
    cls = np.full((H, W), 255); ins = np.zeros((H, W), np.int64); cls[0:16, 0:36] = 15; ins[0:16, 0:36] = 3
    cases["void_in_pred"] = [(pan_image(cls, ins), gt_image(gid), [seg(5, 15, 320)])]
    # prediction mostly over VOID + crowd (ignored) and one just under the threshold (FP)
    gid = np.zeros((H, W), np.int64); gid[:, 24:] = 40; gid[20:, :24] = 41
    cls = np.full((H, W), 255); ins = np.zeros((H, W), np.int64)
    cls[0:10, 16:40] = 16; ins[0:10, 16:40] = 1            # 8 cols void + 16 cols crowd(16) / 24 -> ignored
    cls[10:20, 12:28] = 16; ins[10:20, 12:28] = 2          # 12 cols void + 4 cols crowd: 16/16 -> ignored
    cls[20:32, 0:24] = 16; ins[20:32, 0:24] = 3            # over non-crowd 41 of another category: counted
    cls[20:22, 24:36] = 17; ins[20:22, 24:36] = 4          # over crowd of category 16, category 17: FP
    cases["crowd_ignore"] = [(pan_image(cls, ins), gt_image(gid), [seg(40, 16, 8 * 24 * 1, 1), seg(41, 18, 12 * 24)])]
    # exactly half void + crowd: 0.5 is not > 0.5 -> FP
    gid = np.zeros((H, W), np.int64); gid[:, 24:] = 50; gid[:, 30:] = 51
    cls = np.full((H, W), 255); ins = np.zeros((H, W), np.int64); cls[0:4, 18:30] = 17; ins[0:4, 18:30] = 1
    cases["crowd_half"] = [(pan_image(cls, ins), gt_image(gid), [seg(50, 17, 6 * 32, 1), seg(51, 17, 18 * 32)])]
    # two crowd segments of one category: only the last in table order counts
    for name, order in (("two_crowd_last", (60, 61)), ("two_crowd_first", (61, 60))):
        gid = np.zeros((H, W), np.int64); gid[:, 0:16] = 60; gid[:, 16:32] = 61
        cls = np.full((H, W), 255); ins = np.zeros((H, W), np.int64); cls[:, 10:22] = 18; ins[:, 10:22] = 1
        cls[0:8, 0:8] = 18; ins[0:8, 0:8] = 2
        tab = {60: seg(60, 18, 16 * 32, 1), 61: seg(61, 18, 16 * 32, 1)}
        cases[name] = [(pan_image(cls, ins), gt_image(gid), [tab[order[0]], tab[order[1]]])]
    # ids in the PNG without a table entry; a duplicate id (the later entry wins, with its category and area)
    gid = np.zeros((H, W), np.int64); gid[0:16, :] = 70; gid[16:, :] = 71; gid[16:, 30:] = 72
    cls = np.full((H, W), 5); ins = np.zeros((H, W), np.int64); cls[16:, :] = 13; ins[16:, :] = 9
    cases["missing_ids"] = [(pan_image(cls, ins), gt_image(gid), [seg(70, 5, 16 * 48)])]
    cases["duplicate_id"] = [(pan_image(cls, ins), gt_image(gid),
                              [seg(71, 12, 10), seg(70, 5, 16 * 48), seg(71, 13, 16 * 30), seg(72, 13, 16 * 18)])]
    # table area != pixel count
    cases["table_area"] = [(pan_image(cls, ins), gt_image(gid),
                            [seg(70, 5, 3 * 16 * 48), seg(71, 13, 16 * 30 // 3), seg(72, 13, 16 * 18)])]
    # a stuff class with two instance numbers merges into one segment
    gid = np.zeros((H, W), np.int64); gid[:, :] = 80
    cls = np.full((H, W), 2); ins = np.zeros((H, W), np.int64); ins[:, 24:] = 7
    cases["stuff_merge"] = [(pan_image(cls, ins), gt_image(gid), [seg(80, 2, H * W)])]
    # empty prediction (all void) with segments in the gt; predictions over an all-VOID gt; nothing at all
    gid = np.zeros((H, W), np.int64); gid[:16] = 90; gid[16:] = 91
    cases["empty_pred"] = [(pan_image(np.full((H, W), 255), np.zeros((H, W), np.int64)), gt_image(gid),
                            [seg(90, 1, 16 * 48), seg(91, 11, 16 * 48)])]
    cls = np.full((H, W), 4); ins = np.zeros((H, W), np.int64); cls[:8, :8] = 12; ins[:8, :8] = 3
    cases["void_gt"] = [(pan_image(cls, ins), gt_image(np.zeros((H, W), np.int64)), [])]
    cases["all_void"] = [(pan_image(np.full((H, W), 255), np.zeros((H, W), np.int64)), gt_image(np.zeros((H, W), np.int64)), [])]
    return cases


def noise_mask(rng, H, W, frac, pixel_noise):
    """A boolean mask covering about `frac` of the image: single pixels, or 8x8 blocks."""
    if pixel_noise:
        return rng.random((H, W)) < frac
    return np.kron(rng.random(((H + 7) // 8, (W + 7) // 8)) < frac, np.ones((8, 8), bool))[:H, :W]


def random_image(rng, H, W, n_gt, n_pred_inst, crowd_frac=0.1, void_frac=0.05, pixel_noise=True):
    """A ground truth of ~n_gt rectangles (ids = random, categories random, some crowd, VOID holes) and a prediction
    that perturbs it: shifted boxes, relabelled classes, extra and missing segments, void pixels, 255 instances.
    pixel_noise=False puts the void and the stray stuff instance numbers in small blocks instead of single pixels, which
    keeps a large image small in the compressed fixture."""
    gid = np.zeros((H, W), np.int64)
    cats = {}
    ids = rng.choice(np.arange(1, 1 << 24), n_gt, replace=False)
    stuff_ids = ids[:11]
    band = H // 11 + 1
    for k, i in enumerate(stuff_ids):
        gid[k * band:(k + 1) * band] = i
        cats[int(i)] = k
    cls = np.zeros((H, W), np.int64)
    for k in range(11):
        cls[k * band:(k + 1) * band] = k if rng.random() > 0.15 else (k + 1) % 11
    ins = rng.integers(0, 3, (H, W)) * (noise_mask(rng, H, W, 0.01, pixel_noise))   # stuff pixels with stray instances
    crowd = set()
    for i in ids[11:]:
        h, w = int(rng.integers(4, max(5, H // 6))), int(rng.integers(4, max(5, W // 6)))
        y, x = int(rng.integers(0, H - h)), int(rng.integers(0, W - w))
        c = int(rng.integers(11, 19))
        gid[y:y + h, x:x + w] = i
        cats[int(i)] = c
        if rng.random() < crowd_frac:
            crowd.add(int(i))
    for j in range(n_pred_inst):
        h, w = int(rng.integers(4, max(5, H // 6))), int(rng.integers(4, max(5, W // 6)))
        y, x = int(rng.integers(0, H - h)), int(rng.integers(0, W - w))
        cls[y:y + h, x:x + w] = int(rng.integers(11, 19))
        ins[y:y + h, x:x + w] = 1 + j % 255
    # predictions that copy gt instances (matches), shifted by a few pixels
    for i in ids[11:][: n_gt // 2]:
        ys, xs = np.nonzero(gid == i)
        if ys.size == 0:
            continue
        dy, dx = rng.integers(-2, 3, 2)
        yy, xx = np.clip(ys + dy, 0, H - 1), np.clip(xs + dx, 0, W - 1)
        cls[yy, xx] = cats[int(i)]
        ins[yy, xx] = int(rng.integers(1, 256))
    cls[noise_mask(rng, H, W, void_frac, pixel_noise)] = 255
    gid[noise_mask(rng, H, W, void_frac, pixel_noise)] = 0
    present = set(np.unique(gid).tolist()) - {0}
    segs = []
    for i, c in cats.items():
        if i in present or rng.random() < 0.02:
            segs.append(seg(i, c, int((gid == i).sum()), int(i in crowd)))
    # some ids missing from the table
    drop = rng.random(len(segs)) < 0.03
    segs = [s for s, d in zip(segs, drop) if not d]
    return pan_image(cls, np.minimum(ins, 255)), gt_image(gid), segs


def restore_cases():
    """Label maps from pq_oracle.restore_label (so the tests rebuild them); cv2's output is stored as its sha256 digest."""
    import cv2
    out = []
    for k, (h0, w0, scale, Hp, Wp) in enumerate(((800, 1333, 1024 / 800, 1024, 1728), (800, 1333, 1.6, 1312, 2144),
                                                 (100, 150, 0.6, 64, 96), (97, 131, 0.5, 64, 96), (61, 83, 1 / 0.6, 128, 160),
                                                 (53, 77, 1.0, 64, 96), (33, 47, 0.75, 32, 64))):
        ho, wo = int(np.rint(h0 * scale)), int(np.rint(w0 * scale))
        im_info = np.array([ho, wo, scale], np.float32)
        lab = P.restore_label(Hp, Wp, k)
        sseg = lab.squeeze(0).astype('uint8')[:int(im_info[0]), :int(im_info[1])]          # upsnet_end2end_test.py:265-266
        want = cv2.resize(sseg, None, None, fx=1 / im_info[2], fy=1 / im_info[2], interpolation=cv2.INTER_NEAREST)
        out.append((np.array([Hp, Wp], np.int64), im_info, np.array(want.shape, np.int64), P.digest(want.astype(np.int64))))
    return out


def main():
    ns = load_reference()
    rng = np.random.default_rng(2024)
    out = {"cat_ids": np.array(sorted(CATS), np.int64), "cat_isthing": np.array([CATS[c]['isthing'] for c in sorted(CATS)], np.int64)}
    cases = small_cases(rng)
    cases["multi_image"] = [random_image(rng, 96, 128, 40, 12) for _ in range(3)] + cases["perfect"] + cases["duplicate_id"]
    cases["large"] = [random_image(rng, 1024, 2048, 300, 120, pixel_noise=False)]
    names = sorted(cases)
    for name in names:
        imgs = cases[name]
        stat, summary, per_class, raises = run_reference(ns, imgs, CATS)
        out[name + "/n"] = np.int64(len(imgs))
        for k, (pan, gt, segs) in enumerate(imgs):
            out["%s/%d/pan" % (name, k)] = pan
            out["%s/%d/gt" % (name, k)] = gt
            out["%s/%d/segs" % (name, k)] = np.array([[s["id"], s["category_id"], s["iscrowd"], s["area"]] for s in segs],
                                                     np.int64).reshape(-1, 4)
        out[name + "/stat"] = stat
        out[name + "/summary"] = summary
        out[name + "/per_class"] = per_class
        out[name + "/raises"] = np.int64(raises)
        print("%-16s images %d  tp %3d fp %3d fn %3d  PQ %s" % (name, len(imgs), stat[:, 1].sum(), stat[:, 2].sum(), stat[:, 3].sum(),
                                                                 "ZeroDivisionError" if raises else "%.4f" % summary[0, 0]))
    out["cases"] = np.array(names)
    rc = restore_cases()
    for k, (shape, info, want_shape, want_digest) in enumerate(rc):
        out["restore/%d/shape" % k], out["restore/%d/im_info" % k] = shape, info
        out["restore/%d/want_shape" % k], out["restore/%d/want_sha256" % k] = want_shape, np.array(want_digest)
    out["restore/n"] = np.int64(len(rc))
    np.savez_compressed(os.path.join(HERE, "reference_pq.npz"), **out)


if __name__ == "__main__":
    main()
