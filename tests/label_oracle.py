"""numpy restatement of the panoptic training labels of one image: the label block of the reference's data loaders
(dataset/cityscapes.py:166-189, dataset/coco.py:151-187) and what collate / gt_list_to_blob
(dataset/base_dataset.py:925-976) make of it: seg_gt, seg_gt_4x, mask_gt and seg_roi_gt.

* cv2.resize(INTER_NEAREST) is upsnet_b200.operators.label_restore_index, min(floor(i * (1 / fx)), n - 1) with
  1 / fx and the product in double, and the output size cvRound(n * fx).  With a dsize instead of fx (the 28 x 28
  seg_roi_gt resize), cv2's fx is dsize / n in double.
* cv2.resize copies when the output size equals the input size, whatever the scale; the tables then are the identity.
* im_scale is the Python float im_scales[0] (float64), not the float32 of im_info.
* Pillow's ImageDraw.polygon(xy, outline=1, fill=1) on an 'L' image is `pillow_fill`: the outline is skipped because
  its ink equals the fill's, so only polygon_generic's scanline fill matters.  It is restated from how Pillow 12.2
  draws (pinned against the real Pillow by tests/test_labels_cpu.py):
    - the vertices are truncated toward zero to int;
    - a horizontal edge is one span [xmin, xmax] at its row (an edge whose ends truncate to the same point too: a
      polygon inside one pixel sets that pixel);
    - every other edge has dx = float32(x1 - x0) / (y1 - y0) and meets row y at float32((y - y0) * dx) + x0;
    - rows run over [max(ymin, 0), min(ymax, H)], ymin / ymax over every edge; at row y the non-horizontal edges
      with ymin <= y <= ymax are taken in edge order; an edge ending at y < the polygon's ymax adds its x twice;
    - otherwise, when the row is the edge's ymin or ymax and dx != 0 ("connect discontiguous corners"), the first
      EARLIER edge k (in edge order) that also has an end on row y, dx != 0, roundf(its x) == roundf(x), and that
      spans row r = y - 1 if y is the edge's ymax else y + 1 ends the search; with a the edge's x at r and b edge k's,
      x > a + 1 and x > b + 1 moves x to roundf(max(a, b)) + 1, x < a - 1 and x < b - 1 to roundf(min(a, b)) - 1,
      otherwise x stays;
    - the xs are sorted and each pair fills [ROUND_UP(xa), ROUND_DOWN(xb)], clipped to the canvas: ROUND_UP rounds
      half away from zero and ROUND_DOWN half toward zero, by magnitude (x + 0.5 / x - 0.5 in float32 for x >= 0,
      |x| + 0.5 / |x| - 0.5 in double and negated otherwise).
"""
import hashlib
import math

import numpy as np

from upsnet_b200.operators import label_restore_index

f32 = np.float32


# ------------------------------------------------------------------------------------------------
# cv2 INTER_NEAREST
# ------------------------------------------------------------------------------------------------
def cv_size(n, fx):
    """cv2.resize's output length for a scale: cvRound(n * fx), half to even."""
    return int(np.rint(n * fx))


def nearest_fx(n, fx):
    """Source indices of cv2.resize(fx) along an axis of length n.  cv2 copies the image when the output size equals
    the input's, whatever fx is (2 rows at fx 1.25 stay rows 0, 1, where the rule would give 0, 0)."""
    m = cv_size(n, fx)
    return np.arange(n, dtype=np.int64) if m == n else label_restore_index(m, fx, n)


def nearest_dsize(n, m):
    """Source indices of cv2.resize(dsize = m) along an axis of length n: cv2's scale is m / n in double."""
    return label_restore_index(m, m / float(n), n)


def resize_fx(a, fx):
    return a[nearest_fx(a.shape[0], fx)][:, nearest_fx(a.shape[1], fx)]


# ------------------------------------------------------------------------------------------------
# Pillow's polygon fill
# ------------------------------------------------------------------------------------------------
def _roundf(v):
    """C's roundf: half away from zero."""
    return f32(math.copysign(math.floor(abs(float(v)) + 0.5), float(v)))


def round_up(v):
    """Pillow's ROUND_UP, the first x of a span: floor(float32(v + 0.5)) for v >= 0, else -floor(|v| + 0.5)."""
    v = f32(v)
    return int(math.floor(f32(v + f32(0.5)))) if v >= 0 else -int(math.floor(abs(float(v)) + 0.5))


def round_down(v):
    """Pillow's ROUND_DOWN, the last x of a span: ceil(float32(v - 0.5)) for v >= 0, else -ceil(|v| - 0.5)."""
    v = f32(v)
    return int(math.ceil(f32(v - f32(0.5)))) if v >= 0 else -int(math.ceil(abs(float(v)) - 0.5))


def polygon_edges(xy):
    """[(xmin, xmax, ymin, ymax, dx, x0, y0)] of one polygon's flat coordinate list, after truncation to int."""
    xy = [int(v) for v in xy]               # (int) of the double: toward zero
    n = len(xy) // 2
    pts = [(xy[2 * i], xy[2 * i + 1]) for i in range(n)]
    es = []
    for i in range(n):
        (x0, y0), (x1, y1) = pts[i], pts[(i + 1) % n]
        dx = f32(0) if y0 == y1 else f32(f32(x1 - x0) / f32(y1 - y0))
        es.append((min(x0, x1), max(x0, x1), min(y0, y1), max(y0, y1), dx, x0, y0))
    return es


def _x_at(e, y):
    return f32(f32(f32(y - e[6]) * e[4]) + f32(e[5]))


def row_spans(edges, y):
    """The [a, b] spans (unclipped) that the polygon fill sets on row y."""
    spans = [(e[0], e[1]) for e in edges if e[2] == e[3] and e[2] == y]
    slanted = [e for e in edges if e[2] != e[3]]
    if not slanted:
        return spans
    ymax = max(e[3] for e in edges)
    xx = []
    for i, cur in enumerate(slanted):
        if not cur[2] <= y <= cur[3]:
            continue
        xx.append(_x_at(cur, y))
        if y == cur[3] and y < ymax:
            xx.append(xx[-1])
        elif (y == cur[2] or y == cur[3]) and cur[4] != 0:
            r = y - 1 if y == cur[3] else y + 1
            for oth in slanted[:i]:
                if (y != oth[2] and y != oth[3]) or oth[4] == 0 or _roundf(xx[-1]) != _roundf(_x_at(oth, y)):
                    continue
                if not oth[2] <= r <= oth[3]:
                    continue
                a, b = _x_at(cur, r), _x_at(oth, r)
                if xx[-1] > f32(a + f32(1)) and xx[-1] > f32(b + f32(1)):
                    xx[-1] = f32(_roundf(max(a, b)) + f32(1))
                elif xx[-1] < f32(a - f32(1)) and xx[-1] < f32(b - f32(1)):
                    xx[-1] = f32(_roundf(min(a, b)) - f32(1))
                break
    xx.sort()
    for i in range(1, len(xx), 2):
        spans.append((round_up(xx[i - 1]), round_down(xx[i])))
    return spans


def pillow_fill(canvas, xy):
    """ImageDraw.Draw(Image 'L').polygon(xy, outline=1, fill=1) on a uint8 [H,W] canvas, in place."""
    H, W = canvas.shape
    edges = polygon_edges(xy)
    if not edges:
        return canvas
    y0 = max(min(e[2] for e in edges), 0)
    y1 = min(max(e[3] for e in edges), H - 1)
    for y in range(y0, y1 + 1):
        for a, b in row_spans(edges, y):
            a, b = max(a, 0), min(b, W - 1)
            if a <= b:
                canvas[y, a:b + 1] = 1
    return canvas


# ------------------------------------------------------------------------------------------------
# the labels
# ------------------------------------------------------------------------------------------------
def _pad(a, Hp, Wp):
    out = np.full((a.shape[0], Hp, Wp), 255, np.int64)
    out[:, :a.shape[1], :a.shape[2]] = a
    return out


def _padded(n, stride):
    return int(np.ceil(n / float(stride)) * stride)


def canvas_size(im_shape, im_scale, dataset):
    """(H, W) of the Pillow canvas: int(blob / scale) for Cityscapes, int(np.round(blob / scale)) for COCO."""
    Hb, Wb = im_shape
    if dataset == "cityscapes":
        return int(Hb / im_scale), int(Wb / im_scale)
    return int(np.round(Hb / im_scale)), int(np.round(Wb / im_scale))


def instance_rows(entry, dataset):
    """Row indices of the roidb entry drawn into mask_gt, and of the boxes of seg_roi_gt."""
    cls = np.asarray(entry["gt_classes"])
    crowd = np.asarray(entry["is_crowd"])
    if dataset == "cityscapes":
        return np.arange(len(cls)), np.where(cls > 0)[0]
    return np.where(crowd == 0)[0], np.where((cls > 0) & (crowd == 0))[0]


def roi_boxes(entry, rows, im_scale):
    """np.around(boxes * im_scale).astype(int32) with the degenerate-box +1 fix."""
    b = np.around(np.asarray(entry["boxes"])[rows] * im_scale).astype(np.int32).reshape(-1, 4)
    for i in range(len(b)):
        if b[i][3] == b[i][1]:
            b[i][3] += 1
        if b[i][2] == b[i][0]:
            b[i][2] += 1
    return b


def labels(entry, label_map, im_shape, im_scale, dataset="cityscapes", with_roi=False, mask_size=28, stride=32):
    """-> dict seg_gt int64 [1,Hp,Wp], seg_gt_4x int64 [1,Hp/4,Wp/4], mask_gt int64 [G,Hb_p/4,Wb_p/4] and, with_roi,
    seg_roi_gt int64 [n,M,M] of one roidb entry and its uint8 label map; im_shape the resized image's (h, w)."""
    s = float(im_scale)
    seg = np.asarray(label_map, np.uint8)
    if entry["flipped"]:
        seg = seg[:, ::-1]
    seg = resize_fx(seg, s)
    h, w = seg.shape
    Hp, Wp = _padded(h, stride), _padded(w, stride)
    out = {"seg_gt": _pad(seg[None].astype(np.int64), Hp, Wp),
           "seg_gt_4x": _pad(resize_fx(seg, 0.25)[None].astype(np.int64), int(Hp * 0.25), int(Wp * 0.25))}
    Hb, Wb = im_shape
    Hc, Wc = canvas_size(im_shape, s, dataset)
    if (cv_size(Hc, s), cv_size(Wc, s)) != (Hb, Wb):
        raise ValueError("canvas %dx%d resized by %r is not the blob's %dx%d" % (Hc, Wc, s, Hb, Wb))
    draw, roi_rows = instance_rows(entry, dataset)
    rows, cols = nearest_fx(Hc, s), nearest_fx(Wc, s)
    qrows, qcols = nearest_fx(Hb, 0.25), nearest_fx(Wb, 0.25)
    masks = np.zeros((len(draw), len(qrows), len(qcols)), np.int64)
    for g, i in enumerate(draw):
        canvas = np.zeros((Hc, Wc), np.uint8)
        for p in entry["segms"][i]:
            pillow_fill(canvas, p)
        masks[g] = canvas[rows[qrows]][:, cols[qcols]]
    out["mask_gt"] = _pad(masks, int(_padded(Hb, stride) * 0.25), int(_padded(Wb, stride) * 0.25))
    if with_roi:
        b = roi_boxes(entry, roi_rows, s)
        roi = np.zeros((len(b), mask_size, mask_size), np.int64)
        for i in range(len(b)):
            crop = seg[b[i][1]:b[i][3], b[i][0]:b[i][2]]
            if crop.size == 0:
                raise ValueError("seg_roi_gt: empty crop for box %d" % i)
            roi[i] = crop[nearest_dsize(crop.shape[0], mask_size)][:, nearest_dsize(crop.shape[1], mask_size)]
        out["seg_roi_gt"] = roi
    return out


# ------------------------------------------------------------------------------------------------
# seeded cases
# ------------------------------------------------------------------------------------------------
def label_png(h, w, seed, classes=19):
    """A synthetic uint8 label map from a per-pixel hash: class ids below `classes` and some 255."""
    y, x = np.meshgrid(np.arange(h, dtype=np.uint64), np.arange(w, dtype=np.uint64), indexing="ij")
    with np.errstate(over="ignore"):
        z = (y * np.uint64(0x9E3779B1) + x * np.uint64(0x85EBCA77) + np.uint64(seed) * np.uint64(0xC2B2AE3D))
        z ^= z >> np.uint64(15)
        z *= np.uint64(0x2C1B3C6D)
        z ^= z >> np.uint64(12)
    v = (z % np.uint64(classes + 2)).astype(np.uint8)
    v[v >= classes] = 255
    return v


def star(rng, cx, cy, r, n):
    ang = np.sort(rng.random(n) * 2 * np.pi)
    rr = r * (0.35 + 0.65 * rng.random(n))
    return [float(v) for v in np.stack([cx + rr * np.cos(ang), cy + rr * np.sin(ang)], 1).ravel()]


def random_entry(rng, h0, w0, G, dataset="cityscapes", flipped=False, max_polys=2, max_verts=24):
    """A roidb entry of G polygon instances on an h0 x w0 image, some touching or crossing its border."""
    segms, boxes = [], []
    for _ in range(G):
        r = rng.uniform(2, max(3, min(h0, w0) / 5.0))
        cx, cy = rng.uniform(-r / 2, w0 + r / 2), rng.uniform(-r / 2, h0 + r / 2)
        ps = [star(rng, cx + rng.uniform(-r, r), cy + rng.uniform(-r, r), r, int(rng.integers(3, max_verts + 1)))
              for _ in range(int(rng.integers(1, max_polys + 1)))]
        segms.append(ps)
        a = np.concatenate([np.asarray(p) for p in ps])
        boxes.append([a[0::2].min(), a[1::2].min(), a[0::2].max(), a[1::2].max()])
    boxes = np.asarray(boxes, np.float32).reshape(-1, 4)
    boxes[:, 0::2] = np.clip(boxes[:, 0::2], 0, w0 - 1)             # json_dataset clips the boxes to the image
    boxes[:, 1::2] = np.clip(boxes[:, 1::2], 0, h0 - 1)
    boxes[:, 2:] = np.maximum(boxes[:, 2:], boxes[:, :2])
    cls = rng.integers(1, 9, G).astype(np.int32)
    crowd = np.zeros(G, np.int32)
    if dataset == "coco" and G > 2:
        crowd[int(rng.integers(0, G))] = 1
    return dict(boxes=boxes, gt_classes=cls, is_crowd=crowd, segms=segms, flipped=flipped, height=h0, width=w0)


# the full-size cases: (name, dataset, h0, w0, G, scale, seed); the tests rebuild them and compare sha256 digests
FULL = [("cityscapes_g50", "cityscapes", 1024, 2048, 50, 1.0, 501),
        ("cityscapes_g300", "cityscapes", 1024, 2048, 300, 1.0, 502),
        ("coco_g15", "coco", 480, 800, 15, 800 / 480.0, 503),
        ("coco_g90", "coco", 480, 800, 90, 800 / 480.0, 504)]


def full_case(name):
    _, dataset, h0, w0, G, scale, seed = next(c for c in FULL if c[0] == name)
    rng = np.random.default_rng(seed)
    entry = random_entry(rng, h0, w0, G, dataset, flipped=bool(seed % 2), max_verts=40)
    im_shape = (cv_size(h0, scale), cv_size(w0, scale))
    return entry, label_png(h0, w0, seed), im_shape, scale, dataset


def digest(arrays):
    h = hashlib.sha256()
    for k in sorted(arrays):
        a = np.ascontiguousarray(arrays[k], np.int64)
        h.update(k.encode())
        h.update(str(a.shape).encode())
        h.update(a.tobytes())
    return h.hexdigest()
