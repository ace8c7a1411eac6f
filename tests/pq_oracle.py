"""Test infrastructure: numpy restatements of the reference's label-map restore (upsnet_end2end_test.py:259-266) and of
its per-image PQ statistics (dataset/base_dataset.py:462-608, PQStat.pq_average :73-97).  The oracle of record for the
device kernels on the GPU machine, where the reference does not exist; tests/golden/make_reference_pq.py pins it to the
reference's own code (tests/test_pq_cpu.py).  The product package never imports this module."""
import hashlib

import numpy as np


def restore_label(Hp, Wp, k):
    """Deterministic int64 [1,Hp,Wp] label map for restore case k: a per-pixel integer hash in [-3, 300), so values wrap
    through astype(uint8) and any wrong source index changes the output."""
    y = np.arange(Hp, dtype=np.int64)[:, None]
    x = np.arange(Wp, dtype=np.int64)[None, :]
    v = (y * 73856093) ^ (x * 19349663) ^ ((k + 1) * 83492791)
    v = (v ^ (v >> 13)) * 0x5bd1e995
    return ((v ^ (v >> 15)) % 303 - 3)[None]


def digest(a):
    """sha256 of an array's dtype, shape and bytes (C order)."""
    a = np.ascontiguousarray(a)
    return hashlib.sha256(str(a.dtype).encode() + str(a.shape).encode() + a.tobytes()).hexdigest()


def label_restore(label_map, im_info):
    """Crop [:h,:w], astype(uint8), cv2.resize(fx = fy = 1 / im_info[2], INTER_NEAREST) with the float32 im_info of the
    reference: out size cvRound(h * fx), source index min(floor(y * (1 / fx)), h - 1) in double.  -> int64 [oh, ow]."""
    info = np.asarray(im_info, np.float32).reshape(-1)[:3]
    h, w = int(info[0]), int(info[1])
    fx = float(np.float32(1) / info[2])
    src = np.asarray(label_map)
    src = src.reshape(src.shape[-2:])[:h, :w].astype(np.uint8)
    oh, ow = int(np.rint(h * fx)), int(np.rint(w * fx))
    ifx = 1.0 / fx
    sy = np.minimum(np.floor(np.arange(oh) * ifx).astype(np.int64), h - 1)
    sx = np.minimum(np.floor(np.arange(ow) * ifx).astype(np.int64), w - 1)
    return src[sy][:, sx].astype(np.int64)


def pq_image(pan_2ch, gt_rgb, segments_info, categories, stat=None):
    """_converter_2ch_single_core + _pq_compute_single_core for ONE image, added into `stat` {category: [iou, tp, fp,
    fn]} (returned).  A prediction segment is (class, instance) for a thing class and the class alone for a stuff
    class; class 255 is void.  Matches add their IoU in ascending (gt id, prediction segment) order."""
    stat = {} if stat is None else stat
    isthing = np.zeros(256, bool)
    known = np.zeros(256, bool)
    for c, info in categories.items():
        known[int(c)] = True
        isthing[int(c)] = bool(info['isthing'])
    pan = np.asarray(pan_2ch)
    cls = pan[..., 0].astype(np.int64).ravel()
    inst = pan[..., 1].astype(np.int64).ravel()
    valid = cls != 255
    if (~known[cls[valid]]).any():
        raise KeyError("prediction category not in categories: %s" % sorted(set(cls[valid][~known[cls[valid]]].tolist())))
    pk = cls * 256 + np.where(isthing[cls], inst, 0)
    g = np.asarray(gt_rgb).astype(np.int64).reshape(-1, 3)
    gid = g[:, 0] + 256 * g[:, 1] + 65536 * g[:, 2]
    gt = {int(el['id']): el for el in segments_info}
    pkeys, parea = np.unique(pk[valid], return_counts=True)
    pairs, inter = np.unique(gid[valid] * 65536 + pk[valid], return_counts=True)
    pair_map = {(int(p) // 65536, int(p) % 65536): int(i) for p, i in zip(pairs, inter)}
    area_of = dict(zip(pkeys.tolist(), parea.tolist()))

    def entry(c):
        return stat.setdefault(int(c), [0.0, 0, 0, 0])
    gt_matched, pred_matched = set(), set()
    for (gl, pl), i in pair_map.items():                     # dict order = np.unique order = ascending (gt id, pred)
        if gl not in gt:
            continue
        info = gt[gl]
        if info['iscrowd'] == 1 or info['category_id'] != pl // 256:
            continue
        union = area_of[pl] + info['area'] - i - pair_map.get((0, pl), 0)
        iou = np.float64(i) / np.float64(union)
        if iou > 0.5:
            e = entry(info['category_id'])
            e[0] += float(iou)
            e[1] += 1
            gt_matched.add(gl)
            pred_matched.add(pl)
    crowd = {}
    for gl, info in gt.items():
        if gl in gt_matched:
            continue
        if info['iscrowd'] == 1:
            crowd[info['category_id']] = gl
            continue
        entry(info['category_id'])[3] += 1
    for pl, area in area_of.items():
        if pl in pred_matched:
            continue
        i = pair_map.get((0, pl), 0)
        if pl // 256 in crowd:
            i += pair_map.get((crowd[pl // 256], pl), 0)
        if i / area > 0.5:
            continue
        entry(pl // 256)[2] += 1
    return stat


def pq_average(stat, categories, isthing):
    """PQStat.pq_average (base_dataset.py:73-97) on {category: [iou, tp, fp, fn]}."""
    pq, sq, rq, n = 0, 0, 0, 0
    per_class = {}
    for label, info in categories.items():
        if isthing is not None and isthing != (info['isthing'] == 1):
            continue
        iou, tp, fp, fn = stat.get(label, (0.0, 0, 0, 0))
        if tp + fp + fn == 0:
            per_class[label] = {'pq': 0.0, 'sq': 0.0, 'rq': 0.0}
            continue
        n += 1
        pq_c = iou / (tp + 0.5 * fp + 0.5 * fn)
        sq_c = iou / tp if tp != 0 else 0
        rq_c = tp / (tp + 0.5 * fp + 0.5 * fn)
        per_class[label] = {'pq': pq_c, 'sq': sq_c, 'rq': rq_c, 'iou': iou, 'tp': tp, 'fp': fp, 'fn': fn}
        pq += pq_c
        sq += sq_c
        rq += rq_c
    return {'pq': pq / n, 'sq': sq / n, 'rq': rq / n, 'n': n}, per_class
