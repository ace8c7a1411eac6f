"""Generates tests/golden/reference_labels.npz by EXECUTING the reference's panoptic training labels (build container
only: the reference tree is not present on the GPU box).  Run: python tests/golden/make_reference_labels.py

Executed, unmodified, extracted by AST:
  dataset/cityscapes.py   Cityscapes.__getitem__: its `if config.network.has_fcn_head:` block
  dataset/coco.py         COCODataset.__getitem__: its `if config.network.has_fcn_head:` block
  dataset/base_dataset.py BaseDataset.gt_list_to_blob and BaseDataset.collate (the seg_gt / seg_roi_gt / mask_gt keys)
with the real Pillow (ImageDraw.polygon) and the real cv2 (resize).
Stubs:
  * Image.open: the label PNG, a synthetic uint8 map from a per-pixel hash (tests/label_oracle.label_png);
  * get_image_blob: its blob shape (h, w) and im_scales[0] are passed in (the block reads nothing else of them);
  * mask_util: raises (COCO's non-crowd segmentations here are polygons, as ProposalTargets.pack_roidb requires);
  * config: network.has_fcn_head / has_fpn / has_panoptic_head, rpn_feat_stride (4, 8, 16, 32, 64), mask_size 28,
    train.fcn_with_roi_loss per case.
Fixed zip timestamps: a second run writes identical bytes.
"""
import ast
import collections.abc
import os
import sys
import types
import warnings

import cv2
import numpy as np
import PIL
import torch
from PIL import Image, ImageDraw

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)
import label_oracle as LO  # noqa: E402
from make_reference_rpn_targets import REF, save_npz  # noqa: E402


def _method(path, cls, name):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", SyntaxWarning)          # an invalid escape in a docstring of coco.py
        tree = ast.parse(open(path).read())
    for n in tree.body:
        if isinstance(n, ast.ClassDef) and n.name == cls:
            for m in n.body:
                if isinstance(m, ast.FunctionDef) and m.name == name:
                    return m
    raise KeyError((path, cls, name))


def label_block(path, cls):
    fn = _method(path, cls, "__getitem__")
    stmt = next(s for s in fn.body if isinstance(s, ast.If) and ast.unparse(s.test) == "config.network.has_fcn_head")
    return compile(ast.Module(body=[stmt], type_ignores=[]), path, "exec")


def methods(path, cls, names):
    body = [_method(path, cls, n) for n in names]
    ns = {}
    exec(compile(ast.Module(body=body, type_ignores=[]), path, "exec"), ns)
    return ns


class _MaskUtil:
    def __getattr__(self, name):
        raise AssertionError("mask_util.%s: only polygon segmentations are generated" % name)


def config(with_roi):
    net = types.SimpleNamespace(has_fcn_head=True, has_fpn=True, has_panoptic_head=True, mask_size=28,
                                rpn_feat_stride=(4, 8, 16, 32, 64))
    return types.SimpleNamespace(network=net, train=types.SimpleNamespace(fcn_with_roi_loss=with_roi))


BLOCKS = {"cityscapes": (os.path.join(REF, "dataset", "cityscapes.py"), "Cityscapes",
                         "x/images/a_leftImg8bit.png"),
          "coco": (os.path.join(REF, "dataset", "coco.py"), "coco", "x/images/train2017/a.jpg")}


def run_reference(entry, label_map, im_shape, im_scale, dataset, with_roi):
    path, cls, image = BLOCKS[dataset]
    cfg = config(with_roi)
    img_stub = types.SimpleNamespace(open=lambda p: Image.fromarray(label_map), new=Image.new)
    entry = dict(entry, image=image)
    self = types.SimpleNamespace(phase="train", roidb=[entry])
    ns = {"np": np, "cv2": cv2, "Image": img_stub, "ImageDraw": ImageDraw, "mask_util": _MaskUtil(), "config": cfg,
          "self": self, "index": 0, "im_blob": np.zeros((1, 1) + tuple(im_shape), np.float32),
          "im_scales": [float(im_scale)], "label": {"roidb": entry}}
    exec(label_block(path, cls), ns)
    label = ns["label"]
    base = methods(os.path.join(REF, "dataset", "base_dataset.py"), "BaseDataset", ["gt_list_to_blob", "collate"])
    for f in (base["gt_list_to_blob"], base["collate"]):
        f.__globals__.update({"np": np, "cv2": cv2, "torch": torch, "config": cfg,
                              "Sequence": collections.abc.Sequence})
    ds = types.SimpleNamespace()
    ds.gt_list_to_blob = types.MethodType(base["gt_list_to_blob"], ds)
    ds.collate = types.MethodType(base["collate"], ds)
    keys = ["seg_gt", "mask_gt"] + (["seg_roi_gt"] if with_roi else [])
    blob = ds.collate([{k: label[k] for k in keys}])
    return {k: blob[k].numpy() for k in ["seg_gt", "seg_gt_4x", "mask_gt"] + keys[2:]}


def _poly_px(x, y):
    return [x + 0.2, y + 0.3, x + 0.7, y + 0.4, x + 0.5, y + 0.9]


def cases():
    rng = np.random.default_rng(811)
    out = []

    def add(name, dataset, h0, w0, G, scale, flipped=False, with_roi=True, edit=None, **kw):
        e = LO.random_entry(rng, h0, w0, G, dataset, flipped, **kw)
        if edit:
            edit(e)
        im_shape = (LO.cv_size(h0, scale), LO.cv_size(w0, scale))
        out.append((name, dataset, e, LO.label_png(h0, w0, len(out) + 1), im_shape, scale, with_roi))

    def special(e):
        e["segms"][0] = [LO.star(rng, 20, 15, 8, 7), LO.star(rng, 45, 30, 6, 5), _poly_px(30.0, 40.0)]
        e["segms"][1] = [_poly_px(12.0, 12.0)]                          # a one-pixel polygon
        e["segms"][2] = [list(e["segms"][3][0])]                        # an instance overlapping another
        e["boxes"][4] = [10.2, 20.0, 10.4, 30.0]                        # degenerate seg_roi_gt boxes
        e["boxes"][5] = [5.0, 7.3, 9.0, 7.4]

    add("cs_scale1", "cityscapes", 60, 90, 6, 1.0)
    add("cs_scale05", "cityscapes", 60, 90, 6, 0.5)
    add("cs_scale125_flip", "cityscapes", 60, 88, 6, 1.25, flipped=True)
    add("cs_canvas_mismatch", "cityscapes", 60, 90, 3, 1.25)          # int(112 / 1.25) = 89 -> 111 columns: raises
    add("cs_cvround_int", "cityscapes", 61, 87, 5, 0.7)                 # 61 * 0.7 = 42.7: cvRound 43, int 42
    add("cs_special", "cityscapes", 60, 90, 8, 1.0, edit=special, max_polys=3)
    add("cs_g1", "cityscapes", 50, 70, 1, 1.0)
    add("cs_g300", "cityscapes", 40, 56, 300, 1.0, with_roi=False)
    add("coco_800_480", "coco", 48, 64, 7, 800 / 480.0)
    add("coco_1333_640", "coco", 48, 64, 7, 1333 / 640.0, flipped=True)
    add("coco_scale05_noroi", "coco", 70, 50, 5, 0.5, with_roi=False)
    add("coco_special", "coco", 60, 90, 8, 1.0, edit=special, max_polys=3)
    return out


def pack_entry(prefix, e):
    polys = [p for s in e["segms"] for p in s]
    return {prefix + "boxes": np.asarray(e["boxes"], np.float32), prefix + "gt_classes": e["gt_classes"],
            prefix + "is_crowd": e["is_crowd"], prefix + "flipped": np.array(bool(e["flipped"])),
            prefix + "obj_poly": np.cumsum([0] + [len(s) for s in e["segms"]]).astype(np.int64),
            prefix + "poly_coord": np.cumsum([0] + [len(p) for p in polys]).astype(np.int64),
            prefix + "coords": np.concatenate([np.asarray(p, np.float64) for p in polys])}


def main():
    out = {"pillow_version": np.array(PIL.__version__), "cv2_version": np.array(cv2.__version__)}
    names = []
    for name, dataset, e, lab, im_shape, scale, with_roi in cases():
        try:
            ref = run_reference(e, lab, im_shape, scale, dataset, with_roi)
        except (ValueError, cv2.error) as err:     # the canvas resize is not the blob size, or an empty crop
            print(name, "raises:", err)
            ref = {}
        p = name + "/"
        out.update(pack_entry(p, e))
        out[p + "label_map"] = lab
        out[p + "meta"] = np.array([im_shape[0], im_shape[1], int(with_roi), int(not ref)], np.int64)
        out[p + "scale"] = np.array(scale, np.float64)
        out[p + "dataset"] = np.array(dataset)
        for k, v in ref.items():
            out[p + "out_" + k] = v.astype(np.uint8)
        names.append(name)
    out["cases"] = np.array(names)
    for name, *_ in LO.FULL:
        e, lab, im_shape, scale, dataset = LO.full_case(name)
        ref = run_reference(e, lab, im_shape, scale, dataset, True)
        out["full/" + name] = np.array(LO.digest(ref))
        print(name, {k: v.shape for k, v in ref.items()})
    save_npz(os.path.join(HERE, "reference_labels.npz"), out)


if __name__ == "__main__":
    main()
