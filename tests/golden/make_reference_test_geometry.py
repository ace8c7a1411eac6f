"""Generates tests/golden/reference_test_geometry.npz by EXECUTING the reference's test-phase image path on a list of
original image sizes (build container only: the reference tree is not present on the GPU box).
Run: python tests/golden/make_reference_test_geometry.py

Executed, unmodified, extracted by AST:
  dataset/base_dataset.py   BaseDataset.get_image_blob (COCO's test phase: it reads config.train.scales / train.max_size),
                            prep_im_for_blob, im_list_to_blob
  dataset/cityscapes.py     Cityscapes.get_image_blob (phase 'test': config.test.scales / test.max_size)
  dataset/coco.py,          the `data = {'data': im_blob, 'im_info': ...}` assignment of __getitem__'s test branch
  dataset/cityscapes.py
  upsnet_end2end_test.py    the im_post size argument np.round(im_info[:2] / im_info[2]) (line 256) and the semantic
                            restore loop (lines 258-261: crop, astype(uint8), cv2.resize INTER_NEAREST)
with the real cv2 (imread stubbed to return tests/train_sample_cases.image_bgr, resize real).
Stored per case: the config and original size, im_scales[0], the resized blob shape, the padded blob shape, im_info,
the im_post size and the restored size; for three small cases (BLOBS) also the full padded blob.
Fixed zip timestamps: a second run writes identical bytes.
"""
import ast
import os
import sys
import types

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import train_sample_cases as TS  # noqa: E402
from make_reference_labels import _method  # noqa: E402
from make_reference_rpn_targets import REF, save_npz  # noqa: E402

DS = os.path.join(REF, "dataset")

# (config name, dataset, target size, max_size): the shipped test configurations and two small ones the GPU tests run
CONFIGS = {"coco": ("coco", 800, 1333), "cityscapes": ("cityscapes", 1024, 2048),
           "coco_small": ("coco", 96, 160), "cityscapes_small": ("cityscapes", 128, 256)}
BLOBS = ("small_coco_b", "small_coco_d", "small_coco_e")        # cases whose full padded blob is stored

# (name, config, h, w)
CASES = [
    ("coco_landscape", "coco", 480, 640), ("coco_427x640", "coco", 427, 640), ("coco_portrait", "coco", 640, 427),
    ("coco_square", "coco", 500, 500), ("coco_375x500", "coco", 375, 500),
    ("coco_half", "coco", 802, 640),                # 802 * 1.25 = 1002.5: cvRound gives 1002
    ("coco_cap", "coco", 480, 1000),                # 800 / 480 * 1000 > 1333: capped
    ("coco_elongated", "coco", 200, 1000), ("coco_tall", "coco", 1000, 250),
    ("cs_full", "cityscapes", 1024, 2048), ("cs_half", "cityscapes", 512, 1024), ("cs_600x800", "cityscapes", 600, 800),
    ("cs_cap", "cityscapes", 400, 1200),
    # small COCO-like: 96 / 160
    ("small_coco_a", "coco_small", 64, 90), ("small_coco_b", "coco_small", 64, 100),      # both 96 x 160 padded, im_info differs
    ("small_coco_c", "coco_small", 65, 80),
    ("small_coco_d", "coco_small", 60, 200),                 # capped
    ("small_coco_e", "coco_small", 81, 64),          # 81 * 1.5 = 121.5: cvRound gives 122 ("small_coco_f", "coco_small", 70, 70),
    ("small_coco_g", "coco_small", 115, 112),                # im_post size != restored size
    ("small_coco_h", "coco_small", 104, 176),                # capped, and im_post size != restored size
    # small Cityscapes-like: 128 / 256
    ("small_cs_a", "cityscapes_small", 64, 128), ("small_cs_b", "cityscapes_small", 100, 150),
    ("small_cs_c", "cityscapes_small", 96, 200), ("small_cs_d", "cityscapes_small", 50, 60),
]


def config(dataset, target, max_size):
    net = types.SimpleNamespace(has_fpn=True, rpn_feat_stride=(4, 8, 16, 32, 64), use_caffe_model=True,
                                pixel_means=np.array(TS.PIXEL_MEANS))
    # COCO's test phase reads the train section, Cityscapes' the test section: both carry the size under test here, and
    # the other section a size that would show up if the wrong one were read
    other = types.SimpleNamespace(scales=[target // 2], max_size=max_size // 2)
    own = types.SimpleNamespace(scales=[target], max_size=max_size)
    if dataset == "coco":
        return types.SimpleNamespace(network=net, train=own, test=other)
    return types.SimpleNamespace(network=net, train=other, test=own)


def _bind(ds, path, cls, names, glb):
    for n in names:
        ns = {}
        exec(compile(ast.Module(body=[_method(path, cls, n)], type_ignores=[]), path, "exec"), ns)
        ns[n].__globals__.update(glb)
        setattr(ds, n, types.MethodType(ns[n], ds))


def im_info_assign(path):
    """The test branch's `data = {'data': im_blob, 'im_info': np.array([[im_blob.shape[-2], ...]])}` of __getitem__."""
    for node in ast.walk(ast.parse(open(path).read())):
        if (isinstance(node, ast.Assign) and ast.unparse(node.targets[0]) == "data" and isinstance(node.value, ast.Dict)
                and sorted(ast.literal_eval(k) for k in node.value.keys) == ["data", "im_info"]
                and "im_blob.shape[-2]" in ast.unparse(node.value)):
            return compile(ast.Module(body=[node], type_ignores=[]), path, "exec")
    raise LookupError(path)


def script_parts():
    """upsnet_end2end_test.py: the expression im_post receives as the image size, and the semantic restore loop."""
    path = os.path.join(REF, "upsnet_end2end_test.py")
    tree = ast.parse(open(path).read())
    size = next(n.args[-1] for n in ast.walk(tree)
                if isinstance(n, ast.Call) and isinstance(n.func, ast.Name) and n.func.id == "im_post")
    loop = next(n for n in ast.walk(tree) if isinstance(n, ast.For) and ast.unparse(n.iter) == "enumerate(output['ssegs'])")
    return (compile(ast.Expression(body=size), path, "eval"),
            compile(ast.Module(body=[loop], type_ignores=[]), path, "exec"))


def run_reference(dataset, target, max_size, image):
    cfg = config(dataset, target, max_size)
    glb = {"np": np, "cv2": types.SimpleNamespace(imread=lambda p: image.copy(), resize=cv2.resize,
                                                 INTER_LINEAR=cv2.INTER_LINEAR), "config": cfg}
    ds = types.SimpleNamespace(phase="test")
    base = os.path.join(DS, "base_dataset.py")
    _bind(ds, base, "BaseDataset", ["prep_im_for_blob", "im_list_to_blob"], glb)
    if dataset == "cityscapes":
        _bind(ds, os.path.join(DS, "cityscapes.py"), "Cityscapes", ["get_image_blob"], glb)
        path = os.path.join(DS, "cityscapes.py")
    else:
        _bind(ds, base, "BaseDataset", ["get_image_blob"], glb)
        path = os.path.join(DS, "coco.py")
    entry = {"image": "x.png", "flipped": False}
    np.random.seed(0)
    im_blob, im_scales = ds.get_image_blob([entry])
    ns = {"np": np, "im_blob": im_blob, "im_scales": im_scales}
    exec(im_info_assign(path), ns)
    data = ns["data"]
    padded = ds.im_list_to_blob([data["data"]])            # collate's data blob
    size_expr, restore_loop = script_parts()
    im_info = data["im_info"][0]
    im_post = eval(size_expr, {"np": np, "im_info": im_info})
    rs = {"np": np, "cv2": cv2, "output": {"ssegs": [np.zeros((1,) + padded.shape[2:], np.int64)]},
          "im_infos": data["im_info"], "all_ssegs": []}
    exec(restore_loop, rs)
    return im_scales[0], im_blob.shape[-2:], padded, data["im_info"], im_post, rs["all_ssegs"][0].shape


def main():
    out = {"cv2_version": np.array(cv2.__version__)}
    for name, (dataset, target, max_size) in CONFIGS.items():
        out["config/" + name] = np.array([dataset, str(target), str(max_size)])
    for i, (name, cfg, h, w) in enumerate(CASES):
        dataset, target, max_size = CONFIGS[cfg]
        s, resized, blob, im_info, im_post, restored = run_reference(dataset, target, max_size, TS.image_bgr(h, w, 30 + i))
        p = name + "/"
        out.update({p + "config": np.array(cfg), p + "size": np.array([h, w]), p + "image_seed": np.array(30 + i),
                    p + "im_scale": np.array(s), p + "resized": np.array(resized), p + "padded": np.array(blob.shape[2:]),
                    p + "im_info": im_info, p + "im_post": np.asarray(im_post), p + "restored": np.array(restored)})
        if name in BLOBS:
            out[p + "blob"] = blob
        print(name, (h, w), "scale %.6f" % s, "resized", tuple(resized), "padded", blob.shape[2:], "im_post",
              tuple(im_post), "restored", restored)
    out["cases"] = np.array([c[0] for c in CASES])
    save_npz(os.path.join(HERE, "reference_test_geometry.npz"), out)


if __name__ == "__main__":
    main()
