"""Generates tests/golden/reference_train_sample.npz by EXECUTING the reference's training loader on one roidb entry per
case (build container only: the reference tree is not present on the GPU box).
Run: python tests/golden/make_reference_train_sample.py

Executed, unmodified, extracted by AST:
  dataset/cityscapes.py    Cityscapes.get_image_blob and the `if config.network.has_fcn_head:` block of __getitem__
  dataset/coco.py          the `if config.network.has_fcn_head:` block of COCODataset.__getitem__
  dataset/base_dataset.py  BaseDataset.get_image_blob (COCO's), prep_im_for_blob, im_list_to_blob, gt_list_to_blob,
                           collate
  rpn/assign_anchor.py     add_rpn_blobs: the scale, im_height, im_width and im_info lines of its per-image loop
  dataset/json_dataset.py  extend_with_flipped_entries, with mask/mask_transform.py flip_segms (the flipped entries)
with the real cv2 (imread stubbed, resize real) and the real Pillow (ImageDraw.polygon).  np.random.randint is logged
on its way through, so each case records the seed and the scale index the reference drew under it.
Stubs: cv2.imread returns the synthetic image (tests/train_sample_cases.image_bgr), Image.open the synthetic label map
(tests/label_oracle.label_png); mask_util raises (every segmentation here is a polygon list).
Stored per case: the entries (base and, when flipped, the reference's flipped one), the seeds, the drawn index and
im_scale, im_info and gt_classes exactly, the image blob on a row / column grid (the full blob at 1024x2048 would be
25 MB), sha256 digests of seg_gt, seg_gt_4x, mask_gt and seg_roi_gt (int64), and the key / kind / dtype / shape of every
value collate returned.  The RPN fields are not stored: add_rpn_blobs' two np.random.choice draws have no device
twin (RPNTargets' seeded rule), and tests/golden/reference_rpn_targets.npz covers the rest of that function.
Fixed zip timestamps: a second run writes identical bytes.
"""
import ast
import collections.abc
import os
import sys
import types

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
import train_sample_cases as TS  # noqa: E402
from make_reference_labels import _MaskUtil, _method, label_block  # noqa: E402
from make_reference_rpn_targets import REF, _extract, save_npz  # noqa: E402

DS = os.path.join(REF, "dataset")


def config(dataset):
    c = TS.CONFIGS[dataset]
    net = types.SimpleNamespace(has_fcn_head=True, has_fpn=True, has_panoptic_head=True, has_rpn=True, mask_size=28,
                                rpn_feat_stride=(4, 8, 16, 32, 64), use_caffe_model=True,
                                pixel_means=np.array(TS.PIXEL_MEANS))
    train = types.SimpleNamespace(scales=list(c["scales"]), max_size=c["max_size"], fcn_with_roi_loss=c["with_roi"])
    return types.SimpleNamespace(network=net, train=train)


class _LoggedRandom:
    """np.random with randint logged: the scale index get_image_blob draws."""

    def __init__(self):
        self.drawn = []

    def randint(self, *a, **k):
        v = np.random.randint(*a, **k)
        self.drawn.append(v.copy())
        return v

    def __getattr__(self, name):
        return getattr(np.random, name)


class _Np(types.ModuleType):
    def __init__(self, rnd):
        super().__init__("numpy_logged")
        self.random = rnd

    def __getattr__(self, name):
        return getattr(np, name)


def _bind(ds, path, cls, names, glb):
    for n in names:
        ns = {}
        exec(compile(ast.Module(body=[_method(path, cls, n)], type_ignores=[]), path, "exec"), ns)
        ns[n].__globals__.update(glb)
        setattr(ds, n, types.MethodType(ns[n], ds))


def rpn_info_lines():
    """The per-image loop of add_rpn_blobs cut to its scale / im_height / im_width / im_info assignments."""
    path = os.path.join(REF, "rpn", "assign_anchor.py")
    fn = next(n for n in ast.parse(open(path).read()).body if isinstance(n, ast.FunctionDef) and n.name == "add_rpn_blobs")
    loop = next(s for s in fn.body if isinstance(s, ast.For))
    keep = [s for s in loop.body if isinstance(s, ast.Assign) and ast.unparse(s.targets[0]) in
            ("scale", "im_height", "im_width", "im_info")]
    assert [ast.unparse(s.targets[0]) for s in keep] == ["scale", "im_height", "im_width", "im_info"]
    return compile(ast.Module(body=keep, type_ignores=[]), path, "exec")


def flipped_copy(entry):
    ns = {"np": np}
    exec(_extract(os.path.join(REF, "mask", "mask_transform.py"), {"flip_segms"}), ns)
    jd = {"np": np, "segm_utils": types.SimpleNamespace(flip_segms=ns["flip_segms"])}
    exec(_extract(os.path.join(DS, "json_dataset.py"), {"extend_with_flipped_entries"}), jd)
    roidb = [entry]
    jd["extend_with_flipped_entries"](roidb, None)
    return roidb[1]


def run_reference(dataset, entry, image, label_map, np_seed):
    cfg = config(dataset)
    rnd = _LoggedRandom()
    glb = {"np": _Np(rnd), "cv2": types.SimpleNamespace(imread=lambda p: image.copy(), resize=cv2.resize,
                                                       INTER_LINEAR=cv2.INTER_LINEAR, INTER_NEAREST=cv2.INTER_NEAREST),
           "config": cfg, "torch": torch, "Sequence": collections.abc.Sequence}
    ds = types.SimpleNamespace(phase="train")
    base = os.path.join(DS, "base_dataset.py")
    _bind(ds, base, "BaseDataset", ["prep_im_for_blob", "im_list_to_blob", "gt_list_to_blob", "collate"], glb)
    if dataset == "cityscapes":
        _bind(ds, os.path.join(DS, "cityscapes.py"), "Cityscapes", ["get_image_blob"], glb)
        path, cls, name = os.path.join(DS, "cityscapes.py"), "Cityscapes", "x/images/a_leftImg8bit.png"
    else:
        _bind(ds, base, "BaseDataset", ["get_image_blob"], glb)
        path, cls, name = os.path.join(DS, "coco.py"), "coco", "x/images/train2017/a.jpg"
    entry = dict(entry, image=name)
    np.random.seed(np_seed)
    im_blob, im_scales = ds.get_image_blob([entry])
    (ind,) = rnd.drawn
    rpn = {"np": np, "im_scales": im_scales, "entry": entry, "im_i": 0}
    exec(rpn_info_lines(), rpn)
    data = {"data": im_blob, "im_info": rpn["im_info"]}
    label = {"roidb": {k: entry[k] for k in TS.ROIDB_KEYS if k in entry}}
    ns = {"np": np, "cv2": cv2, "Image": types.SimpleNamespace(open=lambda p: Image.fromarray(label_map), new=Image.new),
          "ImageDraw": ImageDraw, "mask_util": _MaskUtil(), "config": cfg, "self": types.SimpleNamespace(phase="train", roidb=[entry]),
          "index": 0, "im_blob": im_blob, "im_scales": im_scales, "label": label}
    exec(label_block(path, cls), ns)
    data_b, label_b, _ = ds.collate([(data, ns["label"], 0)])
    return int(ind[0]), im_scales[0], data_b, label_b


# (name, dataset, h, w, G, scale index to draw, flipped, entry seed)
CASES = [("cs_800", "cityscapes", 1024, 2048, 6, 0, False, 11),
         ("cs_800_flip", "cityscapes", 1024, 2048, 6, 0, True, 11),
         ("cs_928", "cityscapes", 1024, 2048, 7, 4, False, 12),
         ("cs_928_flip", "cityscapes", 1024, 2048, 7, 4, True, 12),
         ("cs_1024_flip", "cityscapes", 1024, 2048, 5, 7, True, 13),       # 1024 / 1024: scale 1, no resize
         ("coco_800_cap", "coco", 480, 1000, 7, 5, False, 14),            # 800 / 480 * 1000 > 1333: capped
         ("coco_704_pad_flip", "coco", 427, 640, 8, 2, True, 15)]         # 704 x 1055: padded to 704 x 1056


def seed_for(n, want):
    """The first np.random seed under which np.random.randint(0, high=n, size=1) draws `want`."""
    s = 0
    while True:
        np.random.seed(s)
        if int(np.random.randint(0, high=n, size=1)[0]) == want:
            return s
        s += 1


def main():
    out = {"pillow_version": np.array(PIL.__version__), "cv2_version": np.array(cv2.__version__)}
    names = []
    for name, dataset, h, w, G, want, flipped, seed in CASES:
        base = LO.random_entry(np.random.default_rng(seed), h, w, G, dataset)
        entry = flipped_copy(base) if flipped else base
        image, label_map = TS.image_bgr(h, w, seed), LO.label_png(h, w, seed)
        np_seed = seed_for(len(TS.CONFIGS[dataset]["scales"]), want)
        ind, s, data, label = run_reference(dataset, entry, image, label_map, np_seed)
        assert ind == want
        p = name + "/"
        out.update(TS.pack_entry(p + "base/", base))
        out.update(TS.pack_entry(p + "entry/", entry))
        blob = data["data"].numpy()
        ho, wo = (int(v) for v in data["im_info"][0, :2])
        rows, cols = TS.grid(ho, blob.shape[2], 23), TS.grid(wo, blob.shape[3], 29)
        out.update({p + "dataset": np.array(dataset), p + "image_seed": np.array(seed), p + "label_seed": np.array(seed),
                    p + "np_seed": np.array(np_seed), p + "scale_index": np.array(ind), p + "im_scale": np.array(s),
                    p + "im_info": data["im_info"], p + "gt_classes": label["gt_classes"].numpy(),
                    p + "blob_rows": rows, p + "blob_cols": cols, p + "blob": blob[0][:, rows][:, :, cols],
                    p + "data_layout": np.array([TS.layout_row(k, v) for k, v in sorted(data.items())]),
                    p + "label_layout": np.array([TS.layout_row(k, v) for k, v in sorted(label.items())])})
        for k in ("seg_gt", "seg_gt_4x", "mask_gt", "seg_roi_gt"):
            if k in label:
                out[p + "digest/" + k] = np.array(LO.digest({k: label[k].numpy()}))
        names.append(name)
        print(name, "index", ind, "scale", s, "blob", blob.shape, {k: tuple(v.shape) for k, v in label.items()
                                                                   if torch.is_tensor(v)})
    out["cases"] = np.array(names)
    save_npz(os.path.join(HERE, "reference_train_sample.npz"), out)


if __name__ == "__main__":
    main()
