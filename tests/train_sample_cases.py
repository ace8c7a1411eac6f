"""The cases of tests/golden/reference_train_sample.npz (what the reference's loader and collate made of one roidb entry
per case), read back for the CPU and GPU tests of TrainingSample, and the synthetic inputs both sides build."""
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "reference_train_sample.npz")
ROIDB_KEYS = ("boxes", "segms", "seg_areas", "gt_classes", "gt_overlaps", "is_crowd", "box_to_gt_ind_map")
PIXEL_MEANS = (102.9801, 115.9465, 122.7717)
CITYSCAPES = dict(scales=(800, 832, 864, 896, 928, 960, 992, 1024), max_size=2048, with_roi=False)
COCO = dict(scales=(640, 672, 704, 736, 768, 800, 832), max_size=1333, with_roi=True)
CONFIGS = {"cityscapes": CITYSCAPES, "coco": COCO}


def image_bgr(h, w, seed):
    """A synthetic decoded image: uint8 [h,w,3], a smooth wave per channel plus 4 bits of per-pixel hash noise.  Smooth
    like a photograph, so that cv2's float resize, whose rounding is not the device's bit for bit, stays within the
    blob tolerance: on pure noise (neighbours up to 255 apart) it strays up to 1.5e-2 from the rule of upsnet_prep_image
    at 1024x2048, ten times more than on this image."""
    y, x, c = np.meshgrid(np.arange(h, dtype=np.uint64), np.arange(w, dtype=np.uint64), np.arange(3, dtype=np.uint64),
                          indexing="ij")
    with np.errstate(over="ignore"):
        z = (y * np.uint64(0x9E3779B1) + x * np.uint64(0x85EBCA77) + c * np.uint64(0x27D4EB2F)
             + np.uint64(seed) * np.uint64(0xC2B2AE3D))
        z ^= z >> np.uint64(15)
        z *= np.uint64(0x2C1B3C6D)
        z ^= z >> np.uint64(13)
    phase = (seed % 7) + c.astype(np.float64)
    wave = 120 + 100 * np.sin(2 * np.pi * x / 97.0 + phase) * np.cos(2 * np.pi * y / 61.0 + 2 * phase)
    return (wave + (z & np.uint64(15)).astype(np.float64)).astype(np.uint8)


def flip_entry(entry):
    """extend_with_flipped_entries' flipped copy of one entry (json_dataset.py:351-382, mask_transform.py:137-163):
    x -> width - x - 1 for the boxes (x1, x2 swapped) and every polygon vertex."""
    w = entry["width"]
    boxes = np.asarray(entry["boxes"]).copy()
    boxes[:, 0], boxes[:, 2] = w - entry["boxes"][:, 2] - 1, w - entry["boxes"][:, 0] - 1
    segms = []
    for segm in entry["segms"]:
        ps = []
        for p in segm:
            q = np.array(p)
            q[0::2] = w - np.array(p[0::2]) - 1
            ps.append(q.tolist())
        segms.append(ps)
    return dict(entry, boxes=boxes, segms=segms, flipped=True)


def pack_entry(prefix, e):
    polys = [p for s in e["segms"] for p in s]
    return {prefix + "boxes": np.asarray(e["boxes"]), prefix + "gt_classes": e["gt_classes"],
            prefix + "is_crowd": e["is_crowd"], prefix + "flipped": np.array(bool(e["flipped"])),
            prefix + "hw": np.array([e["height"], e["width"]], np.int64),
            prefix + "obj_poly": np.cumsum([0] + [len(s) for s in e["segms"]]).astype(np.int64),
            prefix + "poly_coord": np.cumsum([0] + [len(p) for p in polys]).astype(np.int64),
            prefix + "coords": np.concatenate([np.asarray(p, np.float64) for p in polys])}


def unpack_entry(z, prefix):
    coords, pc, op = z[prefix + "coords"], z[prefix + "poly_coord"], z[prefix + "obj_poly"]
    polys = [[float(v) for v in coords[pc[i]:pc[i + 1]]] for i in range(len(pc) - 1)]
    h, w = (int(v) for v in z[prefix + "hw"])
    return dict(boxes=z[prefix + "boxes"], gt_classes=z[prefix + "gt_classes"], is_crowd=z[prefix + "is_crowd"],
                segms=[polys[op[g]:op[g + 1]] for g in range(len(op) - 1)], flipped=bool(z[prefix + "flipped"]),
                height=h, width=w)


def layout_row(key, v):
    """'key|kind|dtype|shape' of one collated value: kind tensor / ndarray / dict (dict: its sorted keys as dtype)."""
    if isinstance(v, dict):
        return "%s|dict|%s|" % (key, ",".join(sorted(v)))
    kind = "ndarray" if isinstance(v, np.ndarray) else "tensor"
    dt = str(v.dtype).replace("torch.", "")
    return "%s|%s|%s|%s" % (key, kind, dt, ",".join(str(int(s)) for s in v.shape))


def load_cases():
    z = np.load(GOLD)
    out = []
    for name in z["cases"]:
        p = str(name) + "/"
        dataset = str(z[p + "dataset"])
        h, w = (int(v) for v in z[p + "entry/hw"])
        out.append(dict(name=str(name), dataset=dataset, entry=unpack_entry(z, p + "entry/"),
                        base=unpack_entry(z, p + "base/"), image_seed=int(z[p + "image_seed"]),
                        label_seed=int(z[p + "label_seed"]), np_seed=int(z[p + "np_seed"]),
                        scale_index=int(z[p + "scale_index"]), im_scale=z[p + "im_scale"],
                        im_info=z[p + "im_info"], gt_classes=z[p + "gt_classes"],
                        blob_rows=z[p + "blob_rows"], blob_cols=z[p + "blob_cols"], blob=z[p + "blob"],
                        digests={k[len(p) + 7:]: str(z[k]) for k in z.files if k.startswith(p + "digest/")},
                        data_layout=[str(r) for r in z[p + "data_layout"]],
                        label_layout=[str(r) for r in z[p + "label_layout"]], shape=(h, w)))
    return out


def grid(n_valid, n_pad, step):
    """The blob rows (or columns) the fixture keeps: every step-th, plus both sides of the valid / padding edge."""
    keep = set(range(0, n_pad, step)) | {n_valid - 2, n_valid - 1, n_valid, n_pad - 1}
    return np.array(sorted(i for i in keep if 0 <= i < n_pad), np.int64)
