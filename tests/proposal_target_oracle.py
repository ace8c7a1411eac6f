"""numpy restatement of the Mask R-CNN proposal targets of one image (operators/modules/proposal_mask_target.py:37-62):
add_proposals (dataset/json_dataset.py:335-348, 454-516, 538-556), sample_rois (bbox/sample_rois.py:51-176) and
add_mask_rcnn_blobs (mask/mask_transform.py:195-323), with pycocotools' rleFrPoly / rleDecode (cocoapi common/maskApi.c)
restated statement by statement.

* IoU: the compiled bbox.pyx (tests/rpn_target_oracle.iou); first argmax everywhere.
* Draws: np.random.choice is the seeded rule of tests/rpn_target_oracle.choice_positions, stream 0 for the fg draw and
  stream 1 for the bg draw.
* float32 arithmetic follows numpy >= 2 (NEP 50): Python scalars do not widen float32 arrays.
* Two rasterisers: `rle_fr_poly` + `rle_decode` (maskApi.c as written) and `toggle_mask`, the formulation the kernel
  uses (a toggle at column-major index x * M + y for every surviving boundary point, pixel i = XOR of the toggles at
  indices <= i, each edge walked in at most M steps).  tests/test_proposal_targets_cpu.py pins one to the other.
"""
import hashlib
import math
from collections import namedtuple

import numpy as np

import rpn_target_oracle as RO

f32 = np.float32

Config = namedtuple("Config", "num_classes batch_rois fg_fraction fg_thresh bg_hi bg_lo weights M")


def config(**kw):
    """The reference's defaults (config/config.py:45-47, 67, 109-113) with dataset.num_classes = 81 (COCO)."""
    base = dict(num_classes=81, batch_rois=512, fg_fraction=0.25, fg_thresh=0.5, bg_hi=0.5, bg_lo=0.0,
                weights=(10.0, 10.0, 5.0, 5.0), M=28)
    base.update(kw)
    return Config(**base)


# ------------------------------------------------------------------------------------------------
# maskApi.c, as written
# ------------------------------------------------------------------------------------------------
INT_MIN = -(2 ** 31)


def _trunc(a):
    """C's (int) of a double: toward zero (the values stay inside int range here)."""
    return np.trunc(a).astype(np.int64)


def rle_fr_poly(xy, h, w):
    """maskApi.c rleFrPoly(R, xy, k = len(xy) / 2, h, w) -> run lengths (column-major, zeros first)."""
    xy = np.asarray(xy, np.float64)
    k = len(xy) // 2
    scale = 5.0
    x = _trunc(scale * xy[0:2 * k:2] + .5)
    y = _trunc(scale * xy[1:2 * k:2] + .5)
    x = np.append(x, x[0])
    y = np.append(y, y[0])
    us, vs = [], []
    for j in range(k):
        xs, xe, ys, ye = int(x[j]), int(x[j + 1]), int(y[j]), int(y[j + 1])
        dx, dy = abs(xe - xs), abs(ys - ye)
        flip = (dx >= dy and xs > xe) or (dx < dy and ys > ye)
        if flip:
            xs, xe = xe, xs
            ys, ye = ye, ys
        if dx >= dy:
            d = np.arange(dx + 1, dtype=np.int64)
            t = dx - d if flip else d
            us.append(t + xs)
            if dx == 0:
                vs.append(np.array([INT_MIN], np.int64))       # (int)(ys + NaN * 0 + .5) on x86-64: 0/0 is NaN
            else:
                s = (ye - ys) / dx
                vs.append(_trunc(ys + s * t.astype(np.float64) + .5))
        else:
            d = np.arange(dy + 1, dtype=np.int64)
            t = dy - d if flip else d
            vs.append(t + ys)
            s = (xe - xs) / dy
            us.append(_trunc(xs + s * t.astype(np.float64) + .5))
    u = np.concatenate(us)
    v = np.concatenate(vs)
    j = np.flatnonzero(u[1:] != u[:-1]) + 1
    xd = np.where(u[j] < u[j - 1], u[j], u[j] - 1).astype(np.float64)
    xd = (xd + .5) / scale - .5
    ok = (np.floor(xd) == xd) & (xd >= 0) & (xd <= w - 1)
    yd = np.minimum(v[j], v[j - 1]).astype(np.float64)
    yd = (yd + .5) / scale - .5
    yd = np.ceil(np.where(yd < 0, 0.0, np.where(yd > h, float(h), yd)))
    a = (xd[ok].astype(np.int64) * h + yd[ok].astype(np.int64)).tolist()
    a.append(h * w)
    a.sort()
    p = 0
    for i in range(len(a)):
        t_ = a[i]
        a[i] -= p
        p = t_
    b = [a[0]]
    i = 1
    while i < len(a):
        if a[i] > 0:
            b.append(a[i])
            i += 1
        else:
            i += 1
            if i < len(a):
                b[-1] += a[i]
                i += 1
    return b


def rle_decode(counts, h, w):
    """maskApi.c rleDecode -> uint8 [h, w] (the runs fill the column-major order)."""
    vals = np.arange(len(counts)) % 2
    flat = np.repeat(vals.astype(np.uint8), counts)
    assert flat.size == h * w
    return flat.reshape(w, h).T


# ------------------------------------------------------------------------------------------------
# the kernel's formulation: toggles, edge by edge, at most M steps per edge
# ------------------------------------------------------------------------------------------------
def _vert(c):
    """(int)(5 * c + .5) of a double."""
    return int(math.trunc(5.0 * c + .5))


def edge_toggles(X0, Y0, X1, Y1, M):
    """Column-major indices x * M + y toggled by the surviving boundary points of one edge.

    A point survives when u changes between consecutive points and min(u) = 5n + 2 with 0 <= n <= M - 1: within an
    edge u moves by at most one per point, monotonically, so each n is crossed once at most and the crossing is found
    directly (|dx| >= |dy|: u is t + xs) or by bisection on the same double expression (|dx| < |dy|).  Points of
    consecutive edges share the rounded vertex when it is >= 0; when it is negative, both u values are <= 0 and the
    pair is dropped by xd < 0, so edges are independent."""
    out = []
    dx, dy = abs(X1 - X0), abs(Y1 - Y0)

    def toggle(n, yv):
        yd = (float(yv) + .5) / 5.0 - .5
        yd = 0.0 if yd < 0 else (float(M) if yd > M else yd)
        out.append(n * M + int(math.ceil(yd)))

    if dx >= dy:
        if dx == 0:
            return out
        flip = X0 > X1
        xs, ys, ye = (X1, Y1, Y0) if flip else (X0, Y0, Y1)
        s = (ye - ys) / dx
        lo, hi = xs, xs + dx

        def v(t):
            return int(math.trunc(ys + s * t + .5))
        for n in range(max(0, -(-(lo - 2) // 5)), min(M - 1, (hi - 3) // 5) + 1):
            ta = 5 * n + 2 - xs
            toggle(n, min(v(ta), v(ta + 1)))
    else:
        flip = Y0 > Y1
        xs, xe, ys = (X1, X0, Y1) if flip else (X0, X1, Y0)
        s = (xe - xs) / dy

        def u(t):
            return int(math.trunc(xs + s * t + .5))
        u0, u1 = u(0), u(dy)
        lo, hi = min(u0, u1), max(u0, u1)
        for n in range(max(0, -(-(lo - 2) // 5)), min(M - 1, (hi - 3) // 5) + 1):
            xd = 5 * n + 2
            a, b = 0, dy                      # the first t past the crossing: u(t) >= xd + 1 (s > 0) or <= xd (s < 0)
            while b - a > 1:
                m = (a + b) // 2
                if (u(m) >= xd + 1) if s > 0 else (u(m) <= xd):
                    b = m
                else:
                    a = m
            toggle(n, ys + b - 1)
    return out


def toggle_mask(xy, M):
    """One polygon (normalised double coordinates) -> uint8 [M, M] by toggles and a prefix XOR."""
    xy = np.asarray(xy, np.float64)
    k = len(xy) // 2
    X = [_vert(c) for c in xy[0:2 * k:2]]
    Y = [_vert(c) for c in xy[1:2 * k:2]]
    bits = np.zeros(M * M + 1, np.uint8)
    for j in range(k):
        for a in edge_toggles(X[j], Y[j], X[(j + 1) % k], Y[(j + 1) % k], M):
            bits[a] ^= 1
    flat = np.bitwise_xor.accumulate(bits[:M * M])
    return flat.reshape(M, M).T


def rle_mask(xy, M):
    return rle_decode(rle_fr_poly(xy, M, M), M, M)


# ------------------------------------------------------------------------------------------------
# the targets
# ------------------------------------------------------------------------------------------------
def norm_polys(polys, box, M):
    """polys_to_mask_wrt_box's normalisation, float32: ((p - x1) * M) / max(x2 - x1, 1)."""
    box = np.asarray(box, f32)
    w = np.maximum(box[2] - box[0], f32(1))
    h = np.maximum(box[3] - box[1], f32(1))
    out = []
    for poly in polys:
        p = np.array(poly, dtype=f32)
        p[0::2] = (p[0::2] - box[0]) * f32(M) / w
        p[1::2] = (p[1::2] - box[1]) * f32(M) / h
        out.append(p)
    return out


def poly_mask(polys, box, M, raster=rle_mask):
    """[M, M] uint8: the union of the polygons rasterised in the box's frame."""
    m = np.zeros((M, M), np.uint8)
    for p in norm_polys(polys, box, M):
        m |= raster(p, M)
    return m


def polys_to_boxes(polys_gt):
    return np.array([[min(min(p[::2]) for p in poly), min(min(p[1::2]) for p in poly),
                      max(max(p[::2]) for p in poly), max(max(p[1::2]) for p in poly)] for poly in polys_gt],
                    np.float32).reshape(-1, 4)


def box_targets(ex, gt, weights):
    """bbox_transform_inv in float32 with the weights multiplied first."""
    wx, wy, ww, wh = (f32(v) for v in weights)
    ew = ex[:, 2] - ex[:, 0] + f32(1)
    eh = ex[:, 3] - ex[:, 1] + f32(1)
    ecx = ex[:, 0] + f32(.5) * ew
    ecy = ex[:, 1] + f32(.5) * eh
    gw = gt[:, 2] - gt[:, 0] + f32(1)
    gh = gt[:, 3] - gt[:, 1] + f32(1)
    gcx = gt[:, 0] + f32(.5) * gw
    gcy = gt[:, 1] + f32(.5) * gh
    return np.stack([wx * (gcx - ecx) / ew, wy * (gcy - ecy) / eh, ww * np.log(gw / ew), wh * np.log(gh / eh)],
                    1).astype(f32)


def gt_max(entry):
    """Max / first argmax over classes of the entry's gt_overlaps rows (dense or scipy sparse)."""
    o = entry["gt_overlaps"]
    o = o.toarray() if hasattr(o, "toarray") else np.asarray(o)
    return o.max(1).astype(f32), o.argmax(1).astype(np.int64)


def proposal_targets(rois, entry, im_scale, cfg, seed, raster=rle_mask):
    """rois float32 [R,5]; entry: boxes, gt_classes, is_crowd, gt_overlaps, box_to_gt_ind_map, segms; im_scale float32.
    -> the nine outputs of ProposalMaskTarget.forward as numpy arrays, plus counts [n_fg, n_bg, n_mask, 0, n_nongt]."""
    rois = np.asarray(rois, f32)
    im_scale = f32(im_scale)
    boxes_gt = np.asarray(entry["boxes"], f32)
    G = boxes_gt.shape[0]
    cls_gt = np.asarray(entry["gt_classes"]).astype(np.int64)
    # add_proposals
    props = rois[rois[:, 0] == 0, 1:] * (f32(1.0) / im_scale)
    gt_inds = np.flatnonzero(cls_gt > 0)
    o = RO.iou(props, boxes_gt[gt_inds]) if len(props) and len(gt_inds) else np.zeros((len(props), 0), f32)
    arg = o.argmax(1) if o.shape[1] else np.zeros(len(props), np.int64)
    mx = o.max(1) if o.shape[1] else np.zeros(len(props), f32)
    pos = mx > 0
    gmax, gcls = gt_max(entry)
    max_ov = np.concatenate([gmax, np.where(pos, mx, f32(0))]).astype(f32)
    max_cls = np.concatenate([gcls, np.where(pos, cls_gt[gt_inds][arg] if o.shape[1] else 0, 0)]).astype(np.int64)
    b2g = np.concatenate([np.asarray(entry["box_to_gt_ind_map"], np.int64),
                          np.where(pos, gt_inds[arg] if o.shape[1] else -1, -1)])
    all_boxes = np.concatenate([boxes_gt, props]).astype(f32)
    all_cls = np.concatenate([cls_gt, np.zeros(len(props), np.int64)])
    # sample_rois
    fg_per_image = int(np.round(cfg.fg_fraction * cfg.batch_rois))
    fg = np.flatnonzero(max_ov >= f32(cfg.fg_thresh))
    n_fg = min(fg_per_image, fg.size)
    if fg.size:
        fg = fg[RO.choice_positions(seed, fg.size, n_fg, 0)]
    bg = np.flatnonzero((max_ov < f32(cfg.bg_hi)) & (max_ov >= f32(cfg.bg_lo)))
    n_bg = min(cfg.batch_rois - n_fg, bg.size)
    if bg.size:
        bg = bg[RO.choice_positions(seed, bg.size, n_bg, 1)]
    keep = np.append(fg, bg).astype(np.int64)
    labels = max_cls[keep].copy()
    labels[n_fg:] = 0
    sampled = all_boxes[keep]
    K = cfg.num_classes
    n = keep.size
    targets = np.zeros((n, 4 * K), f32)
    inside = np.zeros((n, 4 * K), f32)
    fgr = np.flatnonzero(labels > 0)
    if fgr.size:
        gts = all_boxes[gt_inds[b2g[keep[fgr]]]]
        t = box_targets(sampled[fgr], gts, cfg.weights)
        for i, r in enumerate(fgr):
            targets[r, 4 * labels[r]:4 * labels[r] + 4] = t[i]
            inside[r, 4 * labels[r]:4 * labels[r] + 4] = 1
    outside = (inside > 0).astype(f32)
    out_rois = np.hstack([np.zeros((n, 1), f32), sampled * im_scale]).astype(f32)
    nongt = np.flatnonzero(all_cls[keep] == 0).astype(np.int64)
    # add_mask_rcnn_blobs
    M = cfg.M
    has_mask = (labels > 0).astype(np.uint8)
    poly_inds = np.flatnonzero((cls_gt > 0) & (np.asarray(entry["is_crowd"]) == 0))
    polys_gt = [entry["segms"][i] for i in poly_inds]
    if fgr.size:
        obj = RO.iou(sampled[fgr], polys_to_boxes(polys_gt)).argmax(1)
        mask = np.full((fgr.size, K * M * M), -1, f32)
        for i, r in enumerate(fgr):
            m = poly_mask(polys_gt[obj[i]], sampled[r], M, raster)
            mask[i, labels[r] * M * M:(labels[r] + 1) * M * M] = m.reshape(-1)
        mask_boxes = sampled[fgr]
    else:
        bgr = np.flatnonzero(labels == 0)
        if bgr.size == 0:
            raise IndexError("no fg and no bg rois")
        mask_boxes = sampled[bgr[:1]]
        mask = np.full((1, K * M * M), -1, f32)
        has_mask[0] = 1
    mask_rois = np.hstack([np.zeros((len(mask_boxes), 1), f32), mask_boxes * im_scale]).astype(f32)
    counts = np.array([n_fg, n_bg, len(mask_boxes), 0, nongt.size], np.int32)
    return dict(rois=out_rois, labels=labels.astype(np.int64), bbox_targets=targets, bbox_inside_weights=inside,
                bbox_outside_weights=outside, mask_rois=mask_rois, mask_int32=mask, roi_has_mask=has_mask,
                nongt_inds=nongt, counts=counts)


NAMES = ("rois", "labels", "bbox_targets", "bbox_inside_weights", "bbox_outside_weights", "mask_rois", "mask_int32",
         "roi_has_mask", "nongt_inds")


def dxdy_mask(targets):
    """True on the dx / dy columns of a [n, 4K] target blob (dw / dh go through a log)."""
    return np.broadcast_to(np.arange(targets.shape[1]) % 4 < 2, targets.shape)


def digest(out):
    h = hashlib.sha256()
    for k in NAMES:
        v = np.ascontiguousarray(out[k])
        if k == "bbox_targets":
            v = v[dxdy_mask(v)]
        h.update(k.encode())
        h.update(np.ascontiguousarray(v).tobytes())
    return h.hexdigest()


# ------------------------------------------------------------------------------------------------
# synthetic roidb entries and proposals
# ------------------------------------------------------------------------------------------------
def star_polygon(rng, cx, cy, rx, ry, n):
    a = np.sort(rng.uniform(0, 2 * np.pi, n))
    r = rng.uniform(0.5, 1.0, n)
    return [float(round(v, 2)) for xy in zip(cx + rx * r * np.cos(a), cy + ry * r * np.sin(a)) for v in xy]


def entry_from_objects(boxes, classes, crowd, segms, K):
    """A roidb entry as json_dataset._add_gt_annotations writes it (gt_overlaps dense here)."""
    G = len(classes)
    ov = np.zeros((G, K), f32)
    for i, (c, cr) in enumerate(zip(classes, crowd)):
        if cr:
            ov[i] = -1
        else:
            ov[i, c] = 1
    return dict(boxes=np.asarray(boxes, f32).reshape(-1, 4), gt_classes=np.asarray(classes, np.int32),
                is_crowd=np.asarray(crowd, bool), gt_overlaps=ov, box_to_gt_ind_map=np.arange(G, dtype=np.int32),
                segms=list(segms), seg_areas=np.zeros(G, f32))


def random_entry(rng, H, W, G, K, n_crowd=0, max_parts=3, max_verts=40):
    boxes, classes, crowd, segms = [], [], [], []
    for i in range(G + n_crowd):
        cx, cy = rng.uniform(0, W), rng.uniform(0, H)
        rx = float(np.exp(rng.uniform(np.log(4), np.log(W / 4))))
        ry = rx * float(np.exp(rng.uniform(-0.7, 0.7)))
        if i < G:
            parts = [star_polygon(rng, cx + rng.uniform(-rx, rx) * (j > 0), cy + rng.uniform(-ry, ry) * (j > 0),
                                  rx / (1 + j), ry / (1 + j), int(rng.integers(3, max_verts)))
                     for j in range(int(rng.integers(1, max_parts + 1)))]
            parts = [[min(max(v, 0.0), (W - 1.0) if j % 2 == 0 else (H - 1.0)) for j, v in enumerate(p)] for p in parts]
            b = polys_to_boxes([parts])[0]
            segms.append(parts)
        else:
            b = np.array([cx - rx, cy - ry, cx + rx, cy + ry], f32).clip(0, max(H, W) - 1)
            segms.append({"size": [H, W], "counts": "crowd"})
        boxes.append(b)
        classes.append(int(rng.integers(1, K)))
        crowd.append(int(i >= G))
    perm = rng.permutation(G + n_crowd)
    return entry_from_objects(np.asarray(boxes)[perm], np.asarray(classes)[perm], np.asarray(crowd)[perm],
                              [segms[p] for p in perm], K)


def random_rois(rng, entry, n, H, W, im_scale, jitter_frac=0.5):
    """Proposals as PyramidProposal returns them: float32 [n,5], batch column 0, in the scaled frame; half of them
    jittered gt boxes, so that there are fg rows."""
    b = entry["boxes"]
    nj = int(n * jitter_frac)
    src = b[rng.integers(0, len(b), nj)]
    wh = np.maximum(src[:, 2:] - src[:, :2], 1)
    j = src + rng.normal(0, 0.12, (nj, 4)) * np.concatenate([wh, wh], 1)
    c = np.stack([rng.uniform(0, W, n - nj), rng.uniform(0, H, n - nj)], 1)
    s = np.exp(rng.uniform(np.log(8), np.log(W / 2), (n - nj, 2)))
    r = np.concatenate([j, np.concatenate([c - s / 2, c + s / 2], 1)])
    r[:, 0::2] = r[:, 0::2].clip(0, W - 1)
    r[:, 1::2] = r[:, 1::2].clip(0, H - 1)
    r = (r * im_scale).astype(f32)
    return np.concatenate([np.zeros((n, 1), f32), r[rng.permutation(n)]], 1)


# full-size cases, rebuilt from a seed: (name, K, H, W, im_scale, G, R)
FULL = [("coco_g15", 81, 600, 1000, 800 / 600, 15, 2000), ("coco_g90", 81, 600, 1000, 800 / 600, 90, 2000),
        ("cityscapes_g50", 9, 1024, 2048, 1.0, 50, 2000)]


def full_case(name, seed):
    _, K, H, W, scale, G, R = next(c for c in FULL if c[0] == name)
    rng = np.random.default_rng([seed, G, K])
    e = random_entry(rng, H, W, G, K, n_crowd=2)
    return e, random_rois(rng, e, R, H, W, scale), f32(scale), config(num_classes=K)
