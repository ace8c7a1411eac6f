"""numpy restatement of the RPN training targets of one image (rpn/assign_anchor.py:370-595 add_rpn_blobs /
_get_rpn_blobs, generate_anchors.py:50-206, bbox_transform.py:332-363), chunked over anchors so that the full-size
COCO / Cityscapes fields fit in memory.

* IoU: bbox.pyx's bbox_overlaps as Cython compiles it -- the `+ 1` is a double literal and `float(...)` a double cast, so
  iw = f32(f64(f32(min - max)) + 1.0), the areas are products of such doubles, ua is rounded to float32 from a double sum
  and iou = f32(iw * ih) / ua in float32.
* The two np.random.choice draws follow a seeded rule: candidate position p gets key(s, p) = splitmix64(s ^ p * gamma),
  s = seed for the fg draw and splitmix64(seed) for the bg draw, and a draw of `size` returns the positions of the `size`
  smallest keys.
"""
import hashlib
from collections import namedtuple

import numpy as np

GAMMA = np.uint64(0x9E3779B97F4A7C15)

Config = namedtuple("Config", "strides scale ratios rcnn_stride max_size batch fg_fraction pos neg straddle")


def config(max_size=1333, straddle=0, **kw):
    """The reference's defaults (config/config.py:46-52, 118-124) with train.max_size and rpn_straddle_thresh set."""
    base = dict(strides=(4, 8, 16, 32, 64), scale=8, ratios=(0.5, 1, 2), rcnn_stride=32, max_size=max_size, batch=256,
                fg_fraction=0.5, pos=0.7, neg=0.3, straddle=straddle)
    base.update(kw)
    return Config(**base)


def splitmix64(x):
    x = np.asarray(x, np.uint64)
    with np.errstate(over="ignore"):
        z = x + GAMMA
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def draw_keys(seed, n, stream):
    """Keys of positions 0..n-1; stream 0 is the fg draw, 1 the bg draw."""
    s = np.uint64(seed) if stream == 0 else splitmix64(np.uint64(seed))
    with np.errstate(over="ignore"):
        return splitmix64(s ^ (np.arange(n, dtype=np.uint64) * GAMMA))


def choice_positions(seed, n, size, stream):
    """Positions (ascending) of the `size` smallest keys among n."""
    if size <= 0:
        return np.zeros(0, np.int64)
    k = draw_keys(seed, n, stream)
    return np.sort(np.argpartition(k, size - 1)[:size]).astype(np.int64)


def cell_anchors(stride, size, ratios):
    """generate_anchors.py:50-76 / 156-206 for one stride: float64 [A,4]."""
    def whctrs(a):
        w, h = a[2] - a[0] + 1, a[3] - a[1] + 1
        return w, h, a[0] + 0.5 * (w - 1), a[1] + 0.5 * (h - 1)

    def mk(ws, hs, xc, yc):
        ws, hs = ws[:, None], hs[:, None]
        return np.hstack((xc - 0.5 * (ws - 1), yc - 0.5 * (hs - 1), xc + 0.5 * (ws - 1), yc + 0.5 * (hs - 1)))

    w, h, xc, yc = whctrs(np.array([1, 1, stride, stride]) - 1)
    r = np.array(ratios, np.float64)
    ws = np.round(np.sqrt(w * h / r))
    ratio_anchors = mk(ws, np.round(ws * r), xc, yc)
    scales = np.array([size], np.float64) / stride
    out = []
    for a in ratio_anchors:
        w, h, xc, yc = whctrs(a)
        out.append(mk(w * scales, h * scales, xc, yc))
    return np.vstack(out)


def field_sizes(cfg):
    fpn_max = cfg.rcnn_stride * np.ceil(cfg.max_size / float(cfg.rcnn_stride))
    return [int(np.ceil(fpn_max / float(s))) for s in cfg.strides]


def all_anchors(cfg):
    """Concatenated fields of anchors (level, then (y, x), then a), float32 [N,4], and the field sizes."""
    out = []
    Fs = field_sizes(cfg)
    for s, F in zip(cfg.strides, Fs):
        cell = cell_anchors(s, cfg.scale * s, cfg.ratios)
        sh = np.arange(F) * s
        sx, sy = np.meshgrid(sh, sh)
        shifts = np.stack([sx.ravel(), sy.ravel(), sx.ravel(), sy.ravel()], 1)
        out.append((cell[None] + shifts[:, None]).reshape(-1, 4).astype(np.float32))
    return np.concatenate(out), Fs


def iou(anch, gt):
    """bbox_overlaps(anch [n,4] f32, gt [G,4] f32) -> [n,G] f32, with the compiled extension's mixed precision."""
    f32, f64 = np.float32, np.float64
    iw = ((np.minimum(anch[:, None, 2], gt[None, :, 2]) - np.maximum(anch[:, None, 0], gt[None, :, 0])).astype(f64)
          + 1.0).astype(f32)
    ih = ((np.minimum(anch[:, None, 3], gt[None, :, 3]) - np.maximum(anch[:, None, 1], gt[None, :, 1])).astype(f64)
          + 1.0).astype(f32)
    g_area = (((gt[:, 2] - gt[:, 0]).astype(f64) + 1.0) * ((gt[:, 3] - gt[:, 1]).astype(f64) + 1.0)).astype(f32)
    a_area = ((anch[:, 2] - anch[:, 0]).astype(f64) + 1.0) * ((anch[:, 3] - anch[:, 1]).astype(f64) + 1.0)
    inter = iw * ih
    ua = (a_area[:, None] + g_area[None, :].astype(f64) - inter.astype(f64)).astype(f32)
    ok = (iw > 0) & (ih > 0)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(ok, inter / np.where(ok, ua, f32(1)), f32(0)).astype(f32)


def box_targets(ex, gt):
    """bbox_transform_inv with weights 1, float32."""
    ew = ex[:, 2] - ex[:, 0] + 1.0
    eh = ex[:, 3] - ex[:, 1] + 1.0
    ecx = ex[:, 0] + 0.5 * ew
    ecy = ex[:, 1] + 0.5 * eh
    gw = gt[:, 2] - gt[:, 0] + 1.0
    gh = gt[:, 3] - gt[:, 1] + 1.0
    gcx = gt[:, 0] + 0.5 * gw
    gcy = gt[:, 1] + 0.5 * gh
    return np.stack([(gcx - ecx) / ew, (gcy - ecy) / eh, np.log(gw / ew), np.log(gh / eh)], 1).astype(np.float32)


def to_blobs(per_anchor, Fs, A, width):
    """Anchor-order [N] or [N,4] -> the per-level [1,A,F,F] / [1,4A,F,F] blobs, flattened and concatenated."""
    out, s = [], 0
    for F in Fs:
        n = F * F * A
        v = per_anchor[s:s + n]
        out.append(v.reshape(1, F, F, A * width).transpose(0, 3, 1, 2).ravel())
        s += n
    return np.concatenate(out)


def rpn_targets(gt, im_h, im_w, cfg, seed, chunk=8192):
    """-> dict(labels int64 [N], targets / inside / outside float32 [4N] (blob order), log [(kind, n, size)], info)."""
    gt = np.ascontiguousarray(gt, np.float32).reshape(-1, 4)
    if gt.shape[0] == 0:
        raise ValueError("no ground-truth boxes")
    anchors, Fs = all_anchors(cfg)
    A = len(cfg.ratios)
    N = anchors.shape[0]
    st = cfg.straddle
    if st >= 0:
        inside = np.where((anchors[:, 0] >= -st) & (anchors[:, 1] >= -st) & (anchors[:, 2] < im_w + st)
                          & (anchors[:, 3] < im_h + st))[0]
    else:
        inside = np.arange(N)
    an = anchors[inside]
    ni, G = an.shape[0], gt.shape[0]
    amax = np.empty(ni, np.float32)
    aarg = np.empty(ni, np.int64)
    gmax = np.zeros(G, np.float32)
    for s in range(0, ni, chunk):
        o = iou(an[s:s + chunk], gt)
        aarg[s:s + chunk] = o.argmax(1)
        amax[s:s + chunk] = o[np.arange(o.shape[0]), aarg[s:s + chunk]]
        gmax = np.maximum(gmax, o.max(0))
    pos, neg = np.float32(cfg.pos), np.float32(cfg.neg)
    fg = amax >= pos
    for s in range(0, ni, chunk):
        look = np.flatnonzero(~fg[s:s + chunk]) + s
        if look.size:
            fg[look[(iou(an[look], gt) == gmax[None]).any(1)]] = True
    labels = np.full(ni, -1, np.int32)
    labels[fg] = 1
    log = []
    num_fg = int(cfg.fg_fraction * cfg.batch)
    fg_inds = np.where(labels == 1)[0]
    nf = len(fg_inds)
    if nf > num_fg:
        disable = fg_inds[choice_positions(seed, nf, nf - num_fg, 0)]
        log.append(("array", nf, nf - num_fg))
        labels[disable] = -1
    fg_inds = np.where(labels == 1)[0]
    num_bg = cfg.batch - int(np.sum(labels == 1))
    bg_inds = np.where(amax < neg)[0]
    nb = len(bg_inds)
    relabelled = 0
    if nb > num_bg:
        enable = bg_inds[choice_positions(seed, nb, num_bg, 1)]
        log.append(("int", nb, num_bg))
        relabelled = int(np.sum(labels[enable] == 1))
        labels[enable] = 0
    targets = np.zeros((ni, 4), np.float32)
    targets[fg_inds] = box_targets(an[fg_inds], gt[aarg[fg_inds]])
    inside_w = np.zeros((ni, 4), np.float32)
    inside_w[labels == 1] = 1.0
    outside_w = np.zeros((ni, 4), np.float32)
    num_examples = np.sum(labels >= 0)
    if num_examples:
        outside_w[labels >= 0] = 1.0 / num_examples

    def unmap(v, fill):
        r = np.full((N,) + v.shape[1:], fill, v.dtype)
        r[inside] = v
        return r

    out = dict(labels=to_blobs(unmap(labels, -1).astype(np.int64), Fs, A, 1),
               targets=to_blobs(unmap(targets, 0), Fs, A, 4), inside=to_blobs(unmap(inside_w, 0), Fs, A, 4),
               outside=to_blobs(unmap(outside_w, 0), Fs, A, 4), log=log)
    out["counts"] = np.array([ni, nf, int(np.sum(labels == 1)), int(np.sum(labels == 0))], np.int32)
    out["info"] = dict(fg_subsampled=nf > num_fg, no_negatives=nb <= num_bg, zero_max_box=bool((gmax == 0).any()),
                       relabelled=relabelled > 0, pos_exact=bool((amax == pos).any()), neg_exact=bool((amax == neg).any()),
                       tied_max=bool(any((amax == m).sum() > 1 for m in gmax[gmax > 0])), G=G, N=N, Fs=Fs)
    return out


def gt_from_roidb(entry, im_scale):
    """add_rpn_blobs's boxes: non-crowd entries of a class > 0, float32 boxes times the Python float scale."""
    keep = np.where((entry["gt_classes"] > 0) & (entry["is_crowd"] == 0))[0]
    gt = entry["boxes"][keep, :] * float(im_scale)
    return gt.astype(np.float32), np.round(entry["height"] * im_scale), np.round(entry["width"] * im_scale)


def from_roidb(entry, im_scale, cfg, seed):
    gt, h, w = gt_from_roidb(entry, im_scale)
    return rpn_targets(gt, h, w, cfg, seed)


def level_slices(cfg):
    """(labels slice, coords slice, F) of every level in the concatenated blobs."""
    out, s = [], 0
    A = len(cfg.ratios)
    for F in field_sizes(cfg):
        n = A * F * F
        out.append((slice(s, s + n), slice(4 * s, 4 * (s + n)), F))
        s += n
    return out


def xy_mask(cfg):
    """True on the dx / dy channels of the concatenated [1,4A,F,F] blobs (the exact ones; dw / dh go through a log)."""
    A = len(cfg.ratios)
    m = []
    for F in field_sizes(cfg):
        c = np.arange(4 * A) % 4 < 2
        m.append(np.repeat(c, F * F))
    return np.concatenate(m)


def digest(out, cfg):
    h = hashlib.sha256()
    h.update(np.ascontiguousarray(out["labels"], np.int64).tobytes())
    h.update(np.ascontiguousarray(out["targets"], np.float32)[xy_mask(cfg)].tobytes())
    h.update(np.ascontiguousarray(out["inside"], np.float32).tobytes())
    h.update(np.ascontiguousarray(out["outside"], np.float32).tobytes())
    return h.hexdigest()


# full-size cases, rebuilt from a seed: (name, max_size, entry height, width, im_scale, G)
FULL = [("coco_g15", 1333, 600, 1000, 800 / 600, 15), ("coco_g90", 1333, 600, 1000, 800 / 600, 90),
        ("cityscapes_g50", 2048, 1024, 2048, 1.0, 50), ("cityscapes_g300", 2048, 1024, 2048, 1.0, 300)]


def random_roidb(rng, H, W, G, n_crowd=0, n_bg=0):
    """A roidb entry of G object boxes (float32, integer corners as COCO's json loader makes them) plus crowd / class-0
    entries that add_rpn_blobs filters out."""
    n = G + n_crowd + n_bg
    cx, cy = rng.uniform(0, W, n), rng.uniform(0, H, n)
    w = np.exp(rng.uniform(np.log(8), np.log(W / 2), n))
    h = w * np.exp(rng.uniform(-1, 1, n))
    boxes = np.stack([cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2], 1)
    boxes[:, 0::2] = np.clip(np.round(boxes[:, 0::2]), 0, W - 1)
    boxes[:, 1::2] = np.clip(np.round(boxes[:, 1::2]), 0, H - 1)
    cls = rng.integers(1, 81, n).astype(np.int32)
    crowd = np.zeros(n, np.int32)
    crowd[G:G + n_crowd] = 1
    cls[G + n_crowd:] = 0
    perm = rng.permutation(n)
    return dict(boxes=boxes.astype(np.float32)[perm], gt_classes=cls[perm], is_crowd=crowd[perm], height=H, width=W)


def full_case(name, seed):
    _, max_size, H, W, scale, G = next(c for c in FULL if c[0] == name)
    rng = np.random.default_rng([seed, G, max_size])
    return random_roidb(rng, H, W, G, n_crowd=2, n_bg=1), scale, config(max_size=max_size)
