"""Generates tests/golden/reference_sseg.npz by EXECUTING the reference's own semantic-segmentation evaluation (build
container only: the reference tree is not present on the GPU box).  Run: python tests/golden/make_reference_sseg.py

Executed, unmodified, extracted by AST (the modules themselves pull torch datasets, pycocotools and the config at import):
  dataset/base_dataset.py:806-824  BaseDataset.get_confusion_matrix
  dataset/cityscapes.py:399-514    Cityscapes.get_pallete, evaluate_ssegs, write_segmentation_result (palette PNG)
  dataset/coco.py:225-293          coco.evaluate_ssegs, write_segmentation_result (8-bit PNG)
with real PIL PNG writes and reads in a temporary directory laid out like the datasets (the ground truth is written
there as the 8-bit trainId PNG the loaders open), and, for the network-resolution cases, upsnet_end2end_test.py:265-266's
restore with the real cv2.resize(INTER_NEAREST) and the reference's float32 im_info.

evaluate_ssegs only logs its results.  They are captured through the globals it runs with, without editing it: its `np`
is a proxy that records the argument of np.diag (the accumulated confusion matrix) and `logger` a stub that records the
'%.5f' lines of IU_array and meanIU.

Also stored: PIL's own NEAREST source indices for size pairs (read back from an int32 image of column numbers),
including pairs where floor((x + 0.5) * in / out) disagrees with Pillow.  The 1024x2048 case is rebuilt by the tests from
sseg_oracle.synthetic_case, so only its matrix and log lines are stored.
"""
import ast
import os
import sys
import tempfile
import types
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import sseg_oracle as S  # noqa: E402  (synthetic_case: shared with the tests)
REF = "/root/reference/upsnet"


class RecordingNumpy:
    """numpy for evaluate_ssegs's globals; np.diag's argument is the accumulated confusion matrix."""

    def __init__(self):
        self.diag_args = []

    def __getattr__(self, name):
        return getattr(np, name)

    def diag(self, v, *a, **k):
        self.diag_args.append(np.array(v, copy=True))
        return np.diag(v, *a, **k)


class RecordingLogger:
    def __init__(self):
        self.lines = []

    def info(self, msg):
        self.lines.append(str(msg))


def class_methods(path, cls, names, ns):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", SyntaxWarning)          # the '[\[\]]' pattern of the logged matrix
        tree = ast.parse(open(path).read())
        klass = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == cls)
        nodes = [n for n in klass.body if isinstance(n, ast.FunctionDef) and n.name in names]
        assert sorted(n.name for n in nodes) == sorted(names), (path, [n.name for n in nodes])
        exec(compile(ast.Module(body=nodes, type_ignores=[]), path, "exec"), ns)
    return {n: ns[n] for n in names}


def load_reference(variant, num_classes):
    """A dataset object whose methods are the reference's, with recording np / logger globals."""
    from PIL import Image
    base = class_methods(os.path.join(REF, "dataset", "base_dataset.py"), "BaseDataset", ["get_confusion_matrix"], {"np": np})
    rnp, log = RecordingNumpy(), RecordingLogger()
    config = types.SimpleNamespace(dataset=types.SimpleNamespace(num_seg_classes=num_classes))
    ns = {"np": rnp, "os": os, "Image": Image, "config": config, "logger": log}
    if variant == "cityscapes":
        meth = class_methods(os.path.join(REF, "dataset", "cityscapes.py"), "Cityscapes",
                             ["get_pallete", "evaluate_ssegs", "write_segmentation_result"], ns)
    else:
        meth = class_methods(os.path.join(REF, "dataset", "coco.py"), "coco", ["evaluate_ssegs", "write_segmentation_result"], ns)
    ds = type("Dataset", (), dict(base, **meth))()
    return ds, rnp, log


def run_reference(variant, num_classes, preds, gts):
    """evaluate_ssegs over one image list -> (matrix [C,C] float64, the IU / meanIU log lines)."""
    from PIL import Image
    ds, rnp, log = load_reference(variant, num_classes)
    with tempfile.TemporaryDirectory() as tmp:
        ds.roidb = []
        for k, gt in enumerate(gts):
            if variant == "cityscapes":
                image = os.path.join(tmp, "images", "city", "city_%06d_000019_leftImg8bit.png" % k)
                gt_path = image.replace('images', 'labels').replace('leftImg8bit.png', 'gtFine_labelTrainIds.png')
            else:
                image = os.path.join(tmp, "images", "val2017", "%012d.jpg" % (k + 1))
                gt_path = image.replace('images', 'annotations').replace('val2017', 'panoptic_val2017_semantic_trainid_stff').replace('jpg', 'png')
            os.makedirs(os.path.dirname(gt_path), exist_ok=True)
            Image.fromarray(gt).save(gt_path)
            ds.roidb.append({"image": image})
        with np.errstate(divide="ignore", invalid="ignore"):       # the logged row-normalised matrix divides empty rows
            ds.evaluate_ssegs(preds, os.path.join(tmp, "ssegs"))
    np.set_printoptions()
    assert len(rnp.diag_args) == 1
    first = log.lines.index('IU_array:') + 1
    lines = log.lines[first:first + num_classes + 1]
    assert lines[-1].startswith('meanIU:')
    return rnp.diag_args[0], lines


def cv2_restore(label_map, im_info):
    """upsnet_end2end_test.py:265-266 with the real cv2."""
    import cv2
    sseg = label_map.squeeze(0).astype('uint8')[:int(im_info[0]), :int(im_info[1])]
    return cv2.resize(sseg, None, None, fx=1 / im_info[2], fy=1 / im_info[2], interpolation=cv2.INTER_NEAREST)


def closed_form_disagrees(n_in, n_out):
    return not np.array_equal(S.pil_index(n_in, n_out), np.floor((np.arange(n_out) + 0.5) * (n_in / n_out)).astype(np.int64))


def pil_tables(pairs):
    from PIL import Image
    out = []
    for n_in, n_out in pairs:
        img = Image.fromarray(np.tile(np.arange(n_in, dtype=np.int32), (2, 1)))
        out.append(np.array(img.resize((n_out, 2), Image.NEAREST))[0].astype(np.int64))
    return out


def labels(rng, h, w, num_classes, block=(5, 7), out_of_range=0.0, ignore=0.1):
    """Blocky labels in [0, C) with ignored (255) blocks and, optionally, out-of-range [C, 255) blocks."""
    bh, bw = (h + block[0] - 1) // block[0], (w + block[1] - 1) // block[1]
    b = rng.integers(0, num_classes, (bh, bw))
    u = rng.random((bh, bw))
    b[u < ignore] = 255
    b[(u >= ignore) & (u < ignore + out_of_range)] = rng.integers(num_classes, 255, int(((u >= ignore) & (u < ignore + out_of_range)).sum()))
    return np.kron(b, np.ones(block, np.int64))[:h, :w]


def prediction(rng, gt, h, w, num_classes, alias=0.02, dtype=np.uint8, lo=0, hi=256):
    """gt resized to (h, w) with cv2-free nearest sampling, 20 % of the pixels relabelled, `alias` of them in [lo, hi)."""
    H, W = gt.shape
    p = gt[(np.arange(h) * H) // h][:, (np.arange(w) * W) // w].astype(np.int64)
    p[p >= num_classes] = rng.integers(0, num_classes, int((p >= num_classes).sum()))
    r = rng.random((h, w)) < 0.2
    p[r] = rng.integers(0, num_classes, int(r.sum()))
    m = rng.random((h, w)) < alias
    p[m] = rng.integers(lo, hi, int(m.sum()))
    return p.astype(dtype)


def cases(rng):
    """name -> (variant, C, [pred], [gt], [im_info or None])."""
    out = {}
    H, W = 45, 70          # not powers of two: Pillow's sums round, and some input sizes part from the closed form

    def one(name, ph, pw, variant="cityscapes", C=19, **kw):
        gt = labels(rng, H, W, C, out_of_range=kw.pop("oor", 0.05)).astype(np.uint8)
        out[name] = (variant, C, [prediction(rng, gt, ph, pw, C, **kw)], [gt], [None])

    one("equal", H, W)
    one("smaller_1", H - 1, W - 1)
    one("smaller_2", H - 2, W - 2)
    one("larger_1", H + 1, W + 1)
    one("larger_2", H + 2, W + 2)
    one("nonint", 37, 53)
    one("closed_form_disagrees", next(n for n in range(20, 100) if closed_form_disagrees(n, H)),
        next(n for n in range(20, 140) if closed_form_disagrees(n, W)))
    one("up_2x", H // 2, W // 2)
    one("down_2x", 2 * H, 2 * W)
    one("gt_out_of_range", H, W, oor=0.4)
    one("pred_aliasing", 45, 67, alias=0.4, lo=19, hi=256)
    one("int64_wrap", 51, 61, dtype=np.int64, alias=0.3, lo=-300, hi=600)
    out["all_ignored"] = ("cityscapes", 19, [prediction(rng, labels(rng, H, W, 19), H, W, 19)],
                          [np.full((H, W), 255, np.uint8)], [None])
    gt = labels(rng, H, W, 19, out_of_range=0.05)
    gt[gt == 7] = 8
    p = prediction(rng, gt, H - 3, W + 5, 19, alias=0.0)
    p[p == 7] = 9
    out["class_absent"] = ("cityscapes", 19, [p], [gt.astype(np.uint8)], [None])
    preds, gts = [], []
    for h, w, ph, pw in ((48, 64, 48, 64), (40, 56, 41, 55), (33, 47, 64, 90), (52, 70, 26, 35), (45, 61, 44, 63)):
        g = labels(rng, h, w, 19, out_of_range=0.05).astype(np.uint8)
        gts.append(g)
        preds.append(prediction(rng, g, ph, pw, 19, alias=0.05, dtype=np.int64, lo=-20, hi=300))
    out["five_images"] = ("cityscapes", 19, preds, gts, [None] * 5)
    for name, ph, pw, kw in (("coco_equal", H, W, {}), ("coco_nonint", 29, 91, {}),
                             ("coco_int64", 47, 66, dict(dtype=np.int64, alias=0.3, lo=-300, hi=600))):
        gt = labels(rng, H, W, 133, out_of_range=0.05).astype(np.uint8)
        out[name] = ("coco", 133, [prediction(rng, gt, ph, pw, 133, **kw)], [gt], [None])
    # network resolution: padded int64 map + float32 im_info -> cv2 restore -> evaluate (gt at the original size, and for
    # COCO one pixel off it, which the restored size can be when rint(h * scale) / scale does not return to h)
    for name, variant, C, (h0, w0, scale, Hp, Wp), off in (
            ("netres", "cityscapes", 19, (61, 83, 1 / 0.6, 128, 160), (0, 0)),
            ("netres_coco", "coco", 133, (97, 131, 0.5, 64, 96), (1, -1))):
        ho, wo = int(np.rint(h0 * scale)), int(np.rint(w0 * scale))
        info = np.array([ho, wo, scale], np.float32)
        gt = labels(rng, h0 + off[0], w0 + off[1], C, out_of_range=0.05).astype(np.uint8)
        lab = rng.integers(0, C, (1, Hp, Wp))
        lab[:, :ho, :wo] = prediction(rng, gt, ho, wo, C, dtype=np.int64, alias=0.05, lo=-20, hi=300)
        out[name] = (variant, C, [lab], [gt], [info])
    return out


def main():
    rng = np.random.default_rng(2025)
    out = {}
    all_cases = cases(rng)
    for name, (variant, C, preds, gts, infos) in sorted(all_cases.items()):
        ssegs = [p if info is None else cv2_restore(p, info) for p, info in zip(preds, infos)]
        matrix, lines = run_reference(variant, C, ssegs, gts)
        out[name + "/variant"], out[name + "/C"], out[name + "/n"] = np.array(variant), np.int64(C), np.int64(len(preds))
        for k, (p, g, info) in enumerate(zip(preds, gts, infos)):
            out["%s/%d/pred" % (name, k)], out["%s/%d/gt" % (name, k)] = p, g
            if info is not None:
                out["%s/%d/im_info" % (name, k)] = info
        out[name + "/matrix"], out[name + "/lines"] = matrix, np.array(lines)
        print("%-22s %-10s C=%3d images %d  pixels counted %7d  %s" % (name, variant, C, len(preds), matrix.sum(), lines[-1]))
    out["cases"] = np.array(sorted(all_cases))
    # 1024x2048, rebuilt from sseg_oracle.synthetic_case(0, ...): only the reference's matrix and log lines are stored
    pred, gt = S.synthetic_case(0, 1024, 2048, 19)
    matrix, lines = run_reference("cityscapes", 19, [pred], [gt])
    out["large/matrix"], out["large/lines"] = matrix, np.array(lines)
    print("%-22s %-10s C=%3d images 1  pixels counted %7d  %s" % ("large", "cityscapes", 19, matrix.sum(), lines[-1]))
    # PIL's own NEAREST indices
    prng = np.random.default_rng(7)
    pairs = [(427, 426), (426, 427), (1024, 2048), (2048, 1024), (640, 639), (333, 1000), (1000, 333), (7, 3), (3, 7),
             (64, 64), (1, 5), (5, 1)]
    pairs += [tuple(int(v) for v in prng.integers(1, 2100, 2)) for _ in range(40)]
    pairs += [(n_in, n_out) for n_in, n_out in (tuple(int(v) for v in prng.integers(1, 700, 2)) for _ in range(400))
              if closed_form_disagrees(n_in, n_out)][:12]
    out["pil/pairs"] = np.array(pairs, np.int64)
    tabs = pil_tables(pairs)
    out["pil/tables"] = np.concatenate(tabs)
    print("PIL tables: %d pairs, %d where the closed form disagrees" % (len(pairs), sum(closed_form_disagrees(*p) for p in pairs)))
    np.savez_compressed(os.path.join(HERE, "reference_sseg.npz"), **out)


if __name__ == "__main__":
    main()
