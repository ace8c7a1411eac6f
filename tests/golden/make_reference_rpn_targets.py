"""Generates tests/golden/reference_rpn_targets.npz by EXECUTING the reference's RPN training targets (build container
only: the reference tree is not present on the GPU box).  Run: python tests/golden/make_reference_rpn_targets.py

Executed, unmodified, extracted by AST (the modules themselves import the yaml config and the Cython extensions):
  rpn/assign_anchor.py:370-595     add_rpn_blobs, _get_rpn_blobs
  rpn/generate_anchors.py:41-206   get_field_of_anchors (with its thread-local cache), generate_anchors, unmap,
                                   compute_targets and helpers
  bbox/bbox_transform.py:332-363   bbox_transform_inv
  models/rpn.py:60-92              RPNLoss (on the CPU, for the loss values)
  bbox/bbox.pyx                    bbox_overlaps: cythonized and compiled into a temporary directory at generation time
                                   (nothing of it is kept); the Cython version and the C statements of iw and ua are stored
Stubs:
  * config: the reference defaults with train.max_size / rpn_straddle_thresh set per case;
  * np: a module-global proxy of numpy with the np.float alias and random.choice replaced by the seeded key rule of
    tests/rpn_target_oracle.py (an array argument is the fg draw, an int the bg draw); every call is logged;
  * _threadlocal_foa.cache is cleared between cases (its key omits max_size).
The full-size cases (rpn_target_oracle.FULL) are rebuilt by the tests from a seed; only their sha256 digests are stored,
with the dw / dh targets excluded (np.log is not correctly rounded).  The npz is written with fixed zip timestamps, so a
second run gives identical bytes.
"""
import ast
import glob
import io
import os
import re
import subprocess
import sys
import sysconfig
import tempfile
import types
import zipfile
from collections import defaultdict, namedtuple
import threading

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import rpn_target_oracle as RO  # noqa: E402

REF = "/root/reference/upsnet"


def compile_bbox(tmp):
    import Cython
    src = os.path.join(tmp, "bbox.pyx")
    with open(os.path.join(REF, "bbox", "bbox.pyx")) as f, open(src, "w") as g:
        g.write(f.read())
    subprocess.check_call([sys.executable, "-m", "cython", "-3", src, "-o", os.path.join(tmp, "bbox.c")],
                          stdout=subprocess.DEVNULL)
    csrc = open(os.path.join(tmp, "bbox.c")).read()
    so = os.path.join(tmp, "bbox" + sysconfig.get_config_var("EXT_SUFFIX"))
    subprocess.check_call(["gcc", "-shared", "-fPIC", "-O2", "-fwrapv", "-I", sysconfig.get_paths()["include"], "-I",
                           np.get_include(), "-DNPY_NO_DEPRECATED_API=NPY_1_7_API_VERSION", os.path.join(tmp, "bbox.c"),
                           "-o", so])
    import importlib.util
    spec = importlib.util.spec_from_file_location("bbox", so)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)

    def stmt(var):
        # the first C assignment of a variable of bbox_overlaps_c, whitespace collapsed
        m = re.search(r"__pyx_v_%s = ([^;]*);" % var, csrc)
        return " ".join(m.group(1).split())
    return mod.bbox_overlaps, Cython.__version__, {v: stmt(v) for v in ("box_area", "iw", "ih", "ua")}


class _Random:
    def __init__(self):
        self.seed, self.log = 0, []

    def choice(self, a, size=None, replace=True):
        assert not replace
        if isinstance(a, (int, np.integer)):
            kind, n, arr = "int", int(a), None
        else:
            arr = np.asarray(a)
            kind, n = "array", len(arr)
        size = int(size)
        pos = RO.choice_positions(self.seed, n, size, 0 if kind == "array" else 1)
        self.log.append((kind, n, size))
        return pos if arr is None else arr[pos]

    def __getattr__(self, name):
        return getattr(np.random, name)


class _Np(types.ModuleType):
    def __init__(self, rnd):
        super().__init__("numpy_proxy")
        self.random = rnd
        self.float = float

    def __getattr__(self, name):
        return getattr(np, name)


def _extract(path, names=None, skip_imports=True):
    tree = ast.parse(open(path).read())
    body = []
    for n in tree.body:
        if isinstance(n, (ast.Import, ast.ImportFrom)) and skip_imports:
            continue
        if names is None or (isinstance(n, (ast.FunctionDef, ast.ClassDef)) and n.name in names):
            body.append(n)
    return compile(ast.Module(body=body, type_ignores=[]), path, "exec")


def load_reference(bbox_overlaps):
    rnd = _Random()
    npp = _Np(rnd)
    cfg = types.SimpleNamespace(network=types.SimpleNamespace(), train=types.SimpleNamespace())
    bt = {"np": npp}
    exec(_extract(os.path.join(REF, "bbox", "bbox_transform.py"), {"bbox_transform_inv"}), bt)
    ga = {"np": npp, "threading": threading, "namedtuple": namedtuple, "config": cfg,
          "bbox_transform_inv": bt["bbox_transform_inv"]}
    exec(_extract(os.path.join(REF, "rpn", "generate_anchors.py")), ga)
    aa = {"np": npp, "config": cfg, "bbox_overlaps": bbox_overlaps, "get_field_of_anchors": ga["get_field_of_anchors"],
          "compute_targets": ga["compute_targets"], "unmap": ga["unmap"]}
    exec(_extract(os.path.join(REF, "rpn", "assign_anchor.py"), {"add_rpn_blobs", "_get_rpn_blobs"}), aa)
    import torch.nn as nn
    import torch.nn.functional as F
    from functools import reduce
    rl = {"torch": torch, "nn": nn, "F": F, "reduce": reduce, "np": np, "config": cfg}
    exec(_extract(os.path.join(REF, "models", "rpn.py"), {"RPNLoss"}), rl)
    return types.SimpleNamespace(rnd=rnd, cfg=cfg, foa=ga["_threadlocal_foa"], add_rpn_blobs=aa["add_rpn_blobs"],
                                 RPNLoss=rl["RPNLoss"])


def run_reference(R, entry, scale, cfg, seed):
    c = R.cfg
    c.network.has_fpn = True
    c.network.rpn_feat_stride = tuple(cfg.strides)
    c.network.anchor_scales = (cfg.scale,)
    c.network.anchor_ratios = tuple(cfg.ratios)
    c.network.rcnn_feat_stride = cfg.rcnn_stride
    c.train.max_size = cfg.max_size
    c.train.rpn_batch_size = cfg.batch
    c.train.rpn_fg_fraction = cfg.fg_fraction
    c.train.rpn_positive_overlap = cfg.pos
    c.train.rpn_negative_overlap = cfg.neg
    c.train.rpn_straddle_thresh = cfg.straddle
    if hasattr(R.foa, "cache"):
        R.foa.cache.clear()
    R.rnd.seed, R.rnd.log = seed, []
    blobs = defaultdict(list)
    R.add_rpn_blobs(blobs, [scale], [entry])
    out = {}
    for k, key in (("labels", "rpn_labels_int32_wide"), ("targets", "rpn_bbox_targets_wide"),
                   ("inside", "rpn_bbox_inside_weights_wide"), ("outside", "rpn_bbox_outside_weights_wide")):
        v = [blobs["%s_fpn%d" % (key, s)] for s in cfg.strides]
        out[k] = np.concatenate([x.ravel() for x in v])
        if k == "labels":
            out[k] = out[k].astype(np.int64)            # coco.py:135
    out["log"] = list(R.rnd.log)
    out["im_info"] = blobs["im_info"]
    return out


def ref_loss(R, out, cfg, H, W, seed):
    """RPNLoss on seeded head outputs at the feature sizes of an H x W (padded to 32) image; labels as coco.py gives them."""
    g = torch.Generator().manual_seed(seed)
    A = len(cfg.ratios)
    label, scores, preds = {}, [], []
    for (ls, cs, F), s in zip(RO.level_slices(cfg), cfg.strides):
        h, w = -(-H // s), -(-W // s)
        label["rpn_labels_fpn%d" % s] = torch.from_numpy(out["labels"][ls].reshape(1, A, F, F))
        for k, name in (("targets", "rpn_bbox_targets_fpn%d"), ("inside", "rpn_bbox_inside_weights_fpn%d"),
                        ("outside", "rpn_bbox_outside_weights_fpn%d")):
            label[name % s] = torch.from_numpy(out[k][cs].reshape(1, 4 * A, F, F))
        scores.append(torch.randn((1, A, h, w), generator=g))
        preds.append(torch.randn((1, 4 * A, h, w), generator=g) * 0.5)
    cls, box = R.RPNLoss(cfg.batch)(scores, preds, label)
    return float(cls), float(box)


def iou_sample(bbox_overlaps, rng):
    """Anchors-like and box-like float32 boxes with integer, half-integer and arbitrary corners."""
    def boxes(n):
        kind = rng.integers(0, 3, n)
        c = rng.uniform(0, 200, (n, 2))
        s = rng.uniform(1, 80, (n, 2))
        b = np.concatenate([c - s / 2, c + s / 2], 1)
        b[kind == 0] = np.round(b[kind == 0])
        b[kind == 1] = np.round(b[kind == 1] * 2) / 2
        return b.astype(np.float32)
    a, q = boxes(3000), boxes(200)
    return a, q, bbox_overlaps(a, q)


def rect_roidb(boxes, H, W, classes=None, crowd=None):
    b = np.asarray(boxes, np.float32).reshape(-1, 4)
    n = b.shape[0]
    return dict(boxes=b, gt_classes=np.ones(n, np.int32) if classes is None else np.asarray(classes, np.int32),
                is_crowd=np.zeros(n, np.int32) if crowd is None else np.asarray(crowd, np.int32), height=H, width=W)


def exact_iou_box(anchor, target, rng):
    """A box whose IoU with `anchor` is exactly float32(target) under the compiled rule (integer / half corners)."""
    a = np.asarray(anchor, np.float32)[None]
    for _ in range(200000):
        d = rng.integers(-24, 25, 4) / 2.0
        q = (a[0] + d).astype(np.float32)
        if q[2] <= q[0] or q[3] <= q[1]:
            continue
        if RO.iou(a, q[None])[0, 0] == np.float32(target):
            return q
    raise RuntimeError("no box found")


def small_cases(rng):
    cases = {}
    small = RO.config(max_size=224)
    H, W = 180, 224
    cases["typical"] = (RO.random_roidb(rng, H, W, 8), 1.0, small, 11)
    # boxes that are inside anchors themselves: more than 128 fg candidates
    an, _ = RO.all_anchors(small)
    ins = np.flatnonzero((an[:, 0] >= 0) & (an[:, 1] >= 0) & (an[:, 2] < W) & (an[:, 3] < H))
    pick = an[rng.choice(ins, 160, replace=False)]
    cases["fg_subsample"] = (rect_roidb(pick, H, W), 1.0, small, 12)
    # a 48 x 48 image covered by boxes: fewer bg candidates than num_bg, so no anchor is labelled 0
    cases["no_negatives"] = (rect_roidb([[0, 0, 47, 47], [0, 0, 30, 30], [16, 16, 47, 47], [4, 20, 40, 44]], 48, 48),
                             1.0, small, 13)
    # a box with x2 < x1: IoU 0 with every anchor, so its max is 0 and every anchor with a zero IoU is fg
    cases["zero_max_box"] = (rect_roidb([[20, 30, 90, 100], [60, 60, 58, 58]], H, W), 1.0, small, 14)
    # duplicate boxes and a box centred between anchors: tied maxima, first argmax
    cases["ties"] = (rect_roidb([[40, 40, 71, 71], [40, 40, 71, 71], [100, 60, 131, 91], [2, 2, 33, 33],
                                 [102, 60, 133, 91]], H, W), 1.0, small, 15)
    # IoU exactly float32(0.7) and float32(0.3) with one anchor each
    a7 = an[ins[len(ins) // 3]]
    a3 = an[ins[2 * len(ins) // 3]]
    cases["iou_exact"] = (rect_roidb([exact_iou_box(a7, 0.7, rng), exact_iou_box(a3, 0.3, rng)], H, W), 1.0, small, 16)
    cases["straddle_all"] = (RO.random_roidb(rng, H, W, 6), 1.0, RO.config(max_size=224, straddle=-1), 17)
    cases["straddle_16"] = (RO.random_roidb(rng, H, W, 6), 1.0, RO.config(max_size=224, straddle=16), 18)
    cases["crowd_filtered"] = (RO.random_roidb(rng, H, W, 5, n_crowd=3, n_bg=2), 1.0, small, 19)
    cases["g1"] = (RO.random_roidb(rng, H, W, 1), 1.0, small, 20)
    cases["g1500"] = (RO.random_roidb(rng, H, W, 1500), 1.0, small, 21)
    e = RO.random_roidb(rng, 150, 190, 10)
    e["boxes"] = (e["boxes"] + rng.uniform(0, 1, e["boxes"].shape)).astype(np.float32)
    cases["scaled"] = (e, 224 / 190.0 * 0.97, small, 22)
    cases["coco_like"] = (RO.random_roidb(rng, 300, 400, 20), 600 / 300.0, RO.config(max_size=800), 23)
    return cases


def relabel_case(R, rng):
    """A tiny box whose gt-argmax fg anchor is drawn as a negative: search seeds with the oracle, confirm with the run."""
    cfg = RO.config(max_size=224)
    e = rect_roidb([[50, 50, 53, 53], [120, 40, 170, 110]], 180, 224)
    for seed in range(1, 100000):
        if RO.from_roidb(e, 1.0, cfg, seed)["info"]["relabelled"]:
            return e, 1.0, cfg, seed
    raise RuntimeError("no seed relabels")


def save_npz(path, arrays):
    """np.savez_compressed with fixed zip timestamps, so that identical inputs give identical bytes."""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            info.external_attr = 0o644 << 16
            z.writestr(info, buf.getvalue())


def main():
    tmp = tempfile.mkdtemp()
    try:
        bbox_overlaps, cy_version, c_stmt = compile_bbox(tmp)
    finally:
        for f in glob.glob(os.path.join(tmp, "*")):
            os.remove(f)
        os.rmdir(tmp)
    R = load_reference(bbox_overlaps)
    rng = np.random.default_rng(447)
    out = {"cython_version": np.array(cy_version)}
    for k, v in c_stmt.items():
        out["c_stmt/" + k] = np.array(v)
    a, q, o = iou_sample(bbox_overlaps, rng)
    out["iou/boxes"], out["iou/query"], out["iou/overlaps"] = a, q, o
    cases = small_cases(rng)
    cases["relabelled"] = relabel_case(R, rng)
    names = sorted(cases)
    for name in names:
        entry, scale, cfg, seed = cases[name]
        ref = run_reference(R, entry, scale, cfg, seed)
        mine = RO.from_roidb(entry, scale, cfg, seed)
        info = mine["info"]
        for k in ("boxes", "gt_classes", "is_crowd"):
            out["%s/%s" % (name, k)] = entry[k]
        out[name + "/hw"] = np.array([entry["height"], entry["width"]], np.int64)
        out[name + "/scale"] = np.float64(scale)
        out[name + "/cfg"] = np.array([cfg.max_size, cfg.straddle], np.int64)
        out[name + "/seed"] = np.uint64(seed)
        for k in ("labels", "targets", "inside", "outside"):
            out["%s/%s" % (name, k)] = ref[k]
        out[name + "/log_kind"] = np.array([k == "array" for k, _, _ in ref["log"]], np.int64)
        out[name + "/log_n"] = np.array([n for _, n, _ in ref["log"]], np.int64)
        out[name + "/log_size"] = np.array([s for _, _, s in ref["log"]], np.int64)
        out[name + "/im_info"] = ref["im_info"][0]
        for k in ("fg_subsampled", "no_negatives", "zero_max_box", "relabelled", "pos_exact", "neg_exact", "tied_max"):
            out["%s/flag/%s" % (name, k)] = np.int64(info[k])
        H, W = int(ref["im_info"][0][0]), int(ref["im_info"][0][1])
        out[name + "/loss"] = np.array(ref_loss(R, ref, cfg, H, W, seed), np.float64)
        same = all(np.array_equal(ref[k], mine[k]) for k in ("labels", "inside", "outside"))
        print("%-16s G %4d  N %6d  log %-34s flags %s  oracle %s" % (
            name, info["G"], info["N"], ref["log"], "".join(k[0] for k in info if info[k] is True),
            "==" if same else "!="))
    out["cases"] = np.array(names)
    for name, *_ in RO.FULL:
        entry, scale, cfg = RO.full_case(name, 0)
        ref = run_reference(R, entry, scale, cfg, 5)
        out["full/%s/sha256" % name] = np.array(RO.digest(ref, cfg))
        out["full/%s/log_n" % name] = np.array([n for _, n, _ in ref["log"]], np.int64)
        print("%-16s %s log %s" % (name, out["full/%s/sha256" % name], ref["log"]))
    out["full/seed"] = np.uint64(5)
    save_npz(os.path.join(HERE, "reference_rpn_targets.npz"), out)


if __name__ == "__main__":
    main()
