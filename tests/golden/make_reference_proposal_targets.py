"""Generates tests/golden/reference_proposal_targets.npz by EXECUTING the reference's Mask R-CNN proposal targets (build
container only: the reference tree is not present on the GPU box).  Run: python tests/golden/make_reference_proposal_targets.py

Executed, unmodified, extracted by AST:
  operators/modules/proposal_mask_target.py   ProposalMaskTarget.forward (the nine tensor conversions)
  dataset/json_dataset.py                     add_proposals, _merge_proposal_boxes_into_roidb, _filter_crowd_proposals,
                                              _add_class_assignments, extend_with_flipped_entries (the flipped case)
  bbox/sample_rois.py                         sample_rois, _compute_targets, _expand_bbox_targets
  mask/mask_transform.py                      add_mask_rcnn_blobs, polys_to_boxes, polys_to_mask_wrt_box,
                                              _expand_to_class_specific_mask_targets, flip_segms
  bbox/bbox_transform.py                      bbox_transform_inv
  bbox/bbox.pyx                               bbox_overlaps, compiled at generation time (make_reference_rpn_targets)
Stubs:
  * config: the reference's defaults with dataset.num_classes / train.batch_rois / fg_fraction set per case;
  * npr.choice: the seeded rule of tests/rpn_target_oracle.py, stream 0 at the fg call of sample_rois and stream 1 at
    the bg call (told apart by whether the caller has bound bg_inds yet); every call is logged;
  * pycocotools.mask.frPyObjects / decode: tests/proposal_target_oracle.py's statement-by-statement rleFrPoly and
    rleDecode (pycocotools is not installed here);
  * torch inside the module: the device is the CPU and pin_memory is the identity.
The full-size cases (proposal_target_oracle.FULL) are rebuilt by the tests from a seed; only their sha256 digests are
stored, with the dw / dh targets excluded (np.log is not correctly rounded).  Fixed zip timestamps: a second run
writes identical bytes.
"""
import copy
import os
import sys
import tempfile
import glob
import types

import numpy as np
import scipy.sparse
import torch
from collections import defaultdict

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import proposal_target_oracle as PO  # noqa: E402
import rpn_target_oracle as RO  # noqa: E402
from make_reference_rpn_targets import REF, _extract, compile_bbox, save_npz  # noqa: E402

f32 = np.float32


class _Npr:
    def __init__(self):
        self.seed, self.log = 0, []

    def choice(self, a, size=None, replace=True):
        assert not replace
        stream = 1 if "bg_inds" in sys._getframe(1).f_locals else 0
        arr = np.asarray(a)
        pos = RO.choice_positions(self.seed, len(arr), int(size), stream)
        self.log.append((stream, len(arr), int(size)))
        return arr[pos]


class _MaskUtil:
    @staticmethod
    def frPyObjects(pyobj, h, w):
        assert isinstance(pyobj, list) and len(pyobj[0]) > 4          # the polygon-list branch of frPyObjects
        return [{"size": [h, w], "counts": PO.rle_fr_poly(np.array(p, dtype=np.double), h, w)} for p in pyobj]

    @staticmethod
    def decode(rles):
        return np.stack([PO.rle_decode(r["counts"], *r["size"]) for r in rles], 2)


class _Torch(types.ModuleType):
    """torch for the module body: CPU device, pin_memory the identity."""

    class _Pinned:
        def __init__(self, t):
            self.t = t

        def pin_memory(self):
            return self

        def to(self, *a, **k):
            return self.t

    def __init__(self):
        super().__init__("torch_proxy")
        self.tensor = lambda v, dtype=None, requires_grad=False: _Torch._Pinned(torch.tensor(v, dtype=dtype))
        self.device = lambda *a, **k: torch.device("cpu")
        self.cat = torch.cat

    def __getattr__(self, name):
        return getattr(torch, name)


def load_reference(bbox_overlaps):
    npr = _Npr()
    cfg = types.SimpleNamespace(network=types.SimpleNamespace(), train=types.SimpleNamespace(),
                                dataset=types.SimpleNamespace())
    bt = {"np": np}
    exec(_extract(os.path.join(REF, "bbox", "bbox_transform.py"), {"bbox_transform_inv"}), bt)
    mt = {"np": np, "mask_util": _MaskUtil, "config": cfg, "bbox_overlaps": bbox_overlaps}
    exec(_extract(os.path.join(REF, "mask", "mask_transform.py"),
                  {"add_mask_rcnn_blobs", "polys_to_boxes", "polys_to_mask_wrt_box",
                   "_expand_to_class_specific_mask_targets", "flip_segms"}), mt)
    box_utils = types.SimpleNamespace(bbox_overlaps=bbox_overlaps, bbox_transform_inv=bt["bbox_transform_inv"])
    segm_utils = types.SimpleNamespace(flip_segms=mt["flip_segms"])
    jd = {"np": np, "scipy": scipy, "config": cfg, "box_utils": box_utils, "segm_utils": segm_utils}
    exec(_extract(os.path.join(REF, "dataset", "json_dataset.py"),
                  {"add_proposals", "_merge_proposal_boxes_into_roidb", "_filter_crowd_proposals",
                   "_add_class_assignments", "extend_with_flipped_entries"}), jd)
    sr = {"np": np, "npr": npr, "config": cfg, "bbox_transform_inv": bt["bbox_transform_inv"],
          "add_mask_rcnn_blobs": mt["add_mask_rcnn_blobs"]}
    exec(_extract(os.path.join(REF, "bbox", "sample_rois.py"), {"sample_rois", "_compute_targets",
                                                                 "_expand_bbox_targets"}), sr)
    from torch.nn.modules.module import Module
    pm = {"np": np, "torch": _Torch(), "Module": Module, "add_proposals": jd["add_proposals"],
          "sample_rois": sr["sample_rois"], "defaultdict": defaultdict}
    exec(_extract(os.path.join(REF, "operators", "modules", "proposal_mask_target.py"), {"ProposalMaskTarget"}), pm)
    return types.SimpleNamespace(npr=npr, cfg=cfg, module=pm["ProposalMaskTarget"],
                                 flip=jd["extend_with_flipped_entries"])


def ref_entry(e):
    """The oracle's entry in the reference's own format (sparse gt_overlaps, boolean is_crowd), deep-copied."""
    r = copy.deepcopy(e)
    r["gt_overlaps"] = scipy.sparse.csr_matrix(np.asarray(e["gt_overlaps"], f32))
    r["is_crowd"] = np.asarray(e["is_crowd"], bool)
    return r


def run_reference(R, rois, entry, im_scale, cfg, seed):
    c = R.cfg
    c.network.bbox_reg_weights = tuple(cfg.weights)
    c.network.cls_agnostic_bbox_reg = False
    c.network.has_mask_head = True
    c.network.mask_size = cfg.M
    c.dataset.num_classes = cfg.num_classes
    c.train.batch_rois = cfg.batch_rois
    c.train.fg_fraction = cfg.fg_fraction
    c.train.fg_thresh = cfg.fg_thresh
    c.train.bg_thresh_hi = cfg.bg_hi
    c.train.bg_thresh_lo = cfg.bg_lo
    R.npr.seed, R.npr.log = seed, []
    m = R.module(cfg.num_classes, 1, cfg.batch_rois, cfg.fg_fraction, cfg.M, 0.5)
    im_info = np.array([[0, 0, im_scale]], f32)
    outs = m.forward(torch.from_numpy(np.asarray(rois, f32)), ref_entry(entry), im_info)
    return {k: v.numpy() for k, v in zip(PO.NAMES, outs)}, list(R.npr.log)


# ------------------------------------------------------------------------------------------------
# small cases, one per rule
# ------------------------------------------------------------------------------------------------
def rect_poly(x1, y1, x2, y2):
    return [[x1, y1, x2, y1, x2, y2, x1, y2]]


def rois_of(boxes, im_scale=1.0, batch=None):
    b = np.asarray(boxes, f32).reshape(-1, 4) * f32(im_scale)
    col = np.zeros((len(b), 1), f32) if batch is None else np.asarray(batch, f32).reshape(-1, 1)
    return np.concatenate([col, b], 1).astype(f32)


def small_cases(R, rng):
    cases = {}
    K9 = PO.config(num_classes=9, batch_rois=32)
    e = PO.random_entry(rng, 120, 160, 8, 9, n_crowd=1)
    cases["typical"] = (PO.random_rois(rng, e, 300, 120, 160, 1.25), e, f32(1.25), K9, 31)
    # an fg proposal on a crowd box: it regresses to the crowd box with the crowd's class
    e = PO.entry_from_objects([[10, 10, 60, 50], [70, 20, 120, 90]], [3, 5], [0, 1],
                              [rect_poly(10, 10, 60, 50), {"size": [100, 130], "counts": "x"}], 9)
    cases["fg_on_crowd"] = (rois_of([[71, 21, 119, 88], [12, 11, 58, 49], [0, 60, 30, 99]]), e, f32(1), K9, 32)
    # IoU exactly fg_thresh with one gt, exactly 0 with every gt for another (touching: iw = 0)
    e = PO.entry_from_objects([[20, 20, 59, 59]], [2], [0], [rect_poly(20, 20, 59, 59)], 9)
    cases["iou_exact"] = (rois_of([[20, 20, 59, 39], [60, 20, 90, 59], [0, 0, 10, 10]]), e,
                          f32(1), K9, 33)
    # fewer fg than fg_per_image (8 of 32), too few bg for the rest
    e = PO.random_entry(rng, 80, 80, 3, 9)
    cases["few_fg_few_bg"] = (PO.random_rois(rng, e, 12, 80, 80, 1.0, 0.4), e, f32(1), K9, 34)
    # fg_per_image = round(0.5) = 0: no fg rows at all, the first bg row carries an all -1 mask
    e = PO.random_entry(rng, 80, 80, 2, 9)
    cases["no_fg_fallback"] = (PO.random_rois(rng, e, 10, 80, 80, 1.0), e, f32(1),
                               PO.config(num_classes=9, batch_rois=1, fg_fraction=0.5), 35)
    # two gt with the same box: the first argmax decides the class
    e = PO.entry_from_objects([[30, 30, 70, 70], [30, 30, 70, 70], [5, 5, 25, 25]], [4, 6, 2], [0, 0, 0],
                              [rect_poly(30, 30, 70, 70), rect_poly(32, 32, 68, 68), rect_poly(5, 5, 25, 25)], 9)
    cases["iou_tie"] = (rois_of([[31, 30, 70, 71], [29, 31, 69, 70], [6, 5, 24, 26], [80, 80, 95, 95]]), e, f32(1),
                        K9, 36)
    # the box says object 0, the polygon boxes say object 1
    e = PO.entry_from_objects([[10, 10, 80, 80], [100, 10, 140, 50]], [1, 2], [0, 0],
                              [rect_poly(100, 60, 110, 70), [[12, 12, 78, 12, 78, 78, 12, 78]]], 9)
    cases["mask_argmax_differs"] = (rois_of([[11, 10, 80, 79], [100, 10, 141, 50]]), e, f32(1), K9, 37)
    # an object of three polygons, one of them crossing the roi's edge
    e = PO.entry_from_objects([[10, 10, 90, 90]], [7], [0],
                              [[[10, 10, 40, 12, 35, 45, 12, 40], [50, 50, 90, 55, 88, 90, 52, 85, 60, 70],
                                [30, 60, 45, 62, 40, 95, 28, 90]]], 9)
    cases["multi_polygon"] = (rois_of([[12, 12, 88, 88], [5, 20, 60, 80]]), e, f32(1), K9, 38)
    # a roi 0.4 px wide (x2 - x1 < 1, so w = 1) whose object's polygon reaches 1000 px away: 140 000-point edges
    e = PO.entry_from_objects([[200, 100, 200.5, 160], [0, 0, 30, 30]], [3, 1], [0, 0],
                              [[[200.2, 100, 1200, 130, 1190, 900, 150, 160]], rect_poly(0, 0, 30, 30)], 9)
    cases["far_outside_1px"] = (rois_of([[200.1, 101, 200.5, 160], [0, 0, 29, 31]]), e, f32(1), K9, 39)
    # vertices within an ulp of 5 * c + .5 = integer: normalised coordinates near (2k + 1) / 10
    near = []
    for k_ in range(1, 40, 3):
        c = f32(0.1 * (2 * k_ + 1))
        near += [float(np.nextafter(c, f32(0))), float(c), float(np.nextafter(c, f32(10)))]
    pts = [v * 0.3 for v in near]
    poly = [pts[0], pts[1], pts[5], pts[2], pts[9], pts[12], pts[3], pts[14], pts[20], pts[18], pts[0] + 1, pts[30]]
    e = PO.entry_from_objects([[0, 0, 28, 28]], [5], [0], [[poly]], 9)
    cases["half_boundary"] = (rois_of([[0, 0, 28, 28], [0, 0, 27, 28.5]]), e, f32(1), K9, 40)
    # a roi inside the object (negative normalised coordinates) and one covering its top half (y clamped to M)
    e = PO.entry_from_objects([[20, 20, 100, 100]], [8], [0], [[[20, 20, 100, 25, 95, 100, 25, 96, 60, 60]]], 9)
    cases["negative_and_y_clamp"] = (rois_of([[40, 40, 80, 80], [20, 20, 100, 58], [18, 22, 101, 60]]), e, f32(1),
                                     PO.config(num_classes=9, batch_rois=8, fg_fraction=1.0, fg_thresh=0.3), 41)
    # batch index != 0 rows are not proposals of this image
    e = PO.random_entry(rng, 90, 120, 4, 9)
    r = PO.random_rois(rng, e, 40, 90, 120, 1.0)
    r[::3, 0] = 1
    cases["batch_rows"] = (r, e, f32(1), K9, 42)
    # a flipped entry, made by the reference's extend_with_flipped_entries
    e = PO.random_entry(rng, 90, 120, 5, 9)
    db = [ref_entry(e) | {"width": 120, "height": 90}]
    R.flip(db, None)
    fe = db[1]
    fe = dict(fe, gt_overlaps=fe["gt_overlaps"].toarray())
    cases["flipped"] = (PO.random_rois(rng, fe, 60, 90, 120, 1.1), fe, f32(1.1), K9, 43)
    # COCO-like: 81 classes, 512 rois
    e = PO.random_entry(rng, 240, 320, 12, 81, n_crowd=2)
    cases["coco_like"] = (PO.random_rois(rng, e, 600, 240, 320, 1.5), e, f32(1.5), PO.config(), 44)
    return cases


def pack_entry(name, e, out):
    """Entry arrays and the polygons as flat vertices + offsets (crowd segmentations are not stored)."""
    for k in ("boxes", "gt_classes", "is_crowd", "box_to_gt_ind_map"):
        out["%s/%s" % (name, k)] = np.asarray(e[k])
    out[name + "/gt_overlaps"] = np.asarray(e["gt_overlaps"], f32)
    obj_off, poly_off, verts = [0], [0], []
    for s in e["segms"]:
        if isinstance(s, list):
            for p in s:
                verts += list(p)
                poly_off.append(len(verts) // 2)
            obj_off.append(obj_off[-1] + len(s))
        else:
            obj_off.append(obj_off[-1])
    out[name + "/obj_off"] = np.array(obj_off, np.int64)
    out[name + "/poly_off"] = np.array(poly_off, np.int64)
    out[name + "/verts"] = np.array(verts, np.float64)


def main():
    tmp = tempfile.mkdtemp()
    try:
        bbox_overlaps, _, _ = compile_bbox(tmp)
    finally:
        for f in glob.glob(os.path.join(tmp, "*")):
            os.remove(f)
        os.rmdir(tmp)
    R = load_reference(bbox_overlaps)
    rng = np.random.default_rng(2026)
    out = {}
    cases = small_cases(R, rng)
    for name in sorted(cases):
        rois, e, scale, cfg, seed = cases[name]
        ref, log = run_reference(R, rois, e, scale, cfg, seed)
        mine = PO.proposal_targets(rois, e, scale, cfg, seed)
        pack_entry(name, e, out)
        out[name + "/rois_in"] = rois
        out[name + "/scale"] = f32(scale)
        out[name + "/seed"] = np.uint64(seed)
        out[name + "/cfg"] = np.array([cfg.num_classes, cfg.batch_rois, cfg.M], np.int64)
        out[name + "/cfg_f"] = np.array([cfg.fg_fraction, cfg.fg_thresh, cfg.bg_hi, cfg.bg_lo], np.float64)
        out[name + "/log"] = np.array(log, np.int64).reshape(-1, 3)
        for k in PO.NAMES:
            out["%s/%s" % (name, k)] = ref[k]
        same = all(np.array_equal(ref[k], mine[k]) for k in PO.NAMES if k != "bbox_targets")
        print("%-22s rows %3d fg %3d masks %2d log %-28s oracle %s" % (
            name, len(ref["labels"]), int((ref["labels"] > 0).sum()), len(ref["mask_rois"]), log,
            "==" if same else "!="))
    out["cases"] = np.array(sorted(cases))
    for name, *_ in PO.FULL:
        e, rois, scale, cfg = PO.full_case(name, 0)
        ref, log = run_reference(R, rois, e, scale, cfg, 5)
        out["full/%s/sha256" % name] = np.array(PO.digest(ref))
        out["full/%s/log" % name] = np.array(log, np.int64).reshape(-1, 3)
        print("%-22s %s log %s" % (name, out["full/%s/sha256" % name], log))
    out["full/seed"] = np.uint64(5)
    save_npz(os.path.join(HERE, "reference_proposal_targets.npz"), out)


if __name__ == "__main__":
    main()
