"""Numpy restatement of pycocotools' COCOeval (cocoapi PythonAPI/pycocotools/cocoeval.py, default Params) and of the parts
of COCO.loadRes and maskApi.c it relies on (bbIou, rleIou, rleToBbox, rleArea), for iouType 'bbox' and 'segm'.

pycocotools is not installed here and the reference does not vendor it, so this is pinned to the package's published
algorithm, not to executed code; the functions keep the structure of the published ones (_prepare / computeIoU /
evaluateImg / accumulate / summarize) so that they can be read against it line by line.  Masks are uncompressed RLEs
{'size': [h, w], 'counts': uint32 run lengths}, built on oracle.rle_* (maskApi.c rleEncode / rleFrString).

    E = COCOeval(gt_anns, load_res(results, gt_cat_ids, iou_type), img_ids, cat_ids, iou_type)
    E.evaluate(); E.accumulate(); stats = E.summarize()
"""
import os
import sys
from collections import defaultdict

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import oracle as O  # noqa: E402

IOU_THRS = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
REC_THRS = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
MAX_DETS = [1, 10, 100]
AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
AREA_LBL = ['all', 'small', 'medium', 'large']


def to_rle(seg):
    """COCO.annToRLE for the accepted forms: compressed / uncompressed RLE dict or [H,W] mask -> uncompressed RLE."""
    if isinstance(seg, dict):
        c = seg['counts']
        cnts = O.rle_from_string(c) if isinstance(c, (str, bytes)) else np.asarray(c, np.int64).astype(np.uint32)
        return {'size': [int(seg['size'][0]), int(seg['size'][1])], 'counts': cnts}
    m = np.asarray(seg)
    return {'size': [int(m.shape[0]), int(m.shape[1])], 'counts': O.rle_counts(m != 0)}


def rle_area(R):
    """maskApi.c rleArea: the pixel count of the runs of ones (uint)."""
    return int(np.asarray(R['counts'], np.int64)[1::2].sum())


def rle_to_bbox(R):
    """maskApi.c rleToBbox, statement by statement (a mask spanning several columns gets the full height)."""
    h, w = R['size']
    cnts = [int(c) for c in R['counts']]
    m = (len(cnts) // 2) * 2
    xs, ys, xe, ye, cc = w, h, 0, 0, 0
    if m == 0:
        return [0.0, 0.0, 0.0, 0.0]
    xp = 0
    for j in range(m):
        cc += cnts[j]
        t = cc - j % 2
        y = t % h
        x = (t - y) // h
        if j % 2 == 0:
            xp = x
        elif xp < x:
            ys, ye = 0, h - 1
        xs, xe, ys, ye = min(xs, x), max(xe, x), min(ys, y), max(ye, y)
    return [float(xs), float(ys), float(xe - xs + 1), float(ye - ys + 1)]


def bb_iou(dt, gt, iscrowd):
    """maskApi.c bbIou in double: o[d, g]; ga, da are the boxes' own areas; u = da against a crowd region."""
    o = np.zeros((len(dt), len(gt)))
    for g, G in enumerate(gt):
        ga = G[2] * G[3]
        crowd = bool(iscrowd[g])
        for d, D in enumerate(dt):
            da = D[2] * D[3]
            w = min(D[2] + D[0], G[2] + G[0]) - max(D[0], G[0])
            if w <= 0:
                continue
            h = min(D[3] + D[1], G[3] + G[1]) - max(D[1], G[1])
            if h <= 0:
                continue
            i = w * h
            u = da if crowd else da + ga - i
            o[d, g] = i / u
    return o


def rle_iou(dt, gt, iscrowd):
    """maskApi.c rleIou: the bbIou of the rleToBbox boxes decides which pairs are merged; a merged pair gets integer
    intersection i and union u (or the detection's area against a crowd region), then i / u (0 when i == 0).  The merge
    is done here on decoded masks: the same two integers."""
    o = bb_iou([rle_to_bbox(R) for R in dt], [rle_to_bbox(R) for R in gt], iscrowd)
    dec = {}

    def mask(R):
        if id(R) not in dec:
            dec[id(R)] = O.rle_decode(R['counts'], R['size'][0], R['size'][1]).astype(bool)
        return dec[id(R)]
    for g in range(len(gt)):
        for d in range(len(dt)):
            if not o[d, g] > 0:
                continue
            if dt[d]['size'] != gt[g]['size']:
                o[d, g] = -1
                continue
            a, b = mask(dt[d]), mask(gt[g])
            i = int(np.count_nonzero(a & b))
            u = int(np.count_nonzero(a | b))
            if i == 0:
                u = 1
            elif iscrowd[g]:
                u = rle_area(dt[d])
            o[d, g] = float(i) / float(u)
    return o


def load_res(results, iou_type):
    """COCO.loadRes on a results list: ids 1.., iscrowd 0, area = w * h of the result's bbox ('bbox') or the RLE area
    ('segm')."""
    anns = []
    for id_, r in enumerate(results):
        ann = dict(r)
        if iou_type == 'bbox':
            bb = ann['bbox']
            ann['area'] = bb[2] * bb[3]
        else:
            ann['segmentation'] = to_rle(ann['segmentation'])
            ann['area'] = rle_area(ann['segmentation'])
        ann['id'] = id_ + 1
        ann['iscrowd'] = 0
        anns.append(ann)
    return anns


class COCOeval:
    def __init__(self, gts, dts, img_ids, cat_ids, iou_type):
        """gts: ground-truth annotations (image_id, category_id, iscrowd, area, bbox / segmentation, id), in file order;
        dts: load_res output."""
        self.gts_all, self.dts_all, self.iouType = gts, dts, iou_type
        self.imgIds = sorted(set(img_ids))
        self.catIds = sorted(cat_ids)

    def _prepare(self):
        self._gts = defaultdict(list)
        self._dts = defaultdict(list)
        for gt in self.gts_all:
            gt = dict(gt)
            if self.iouType == 'segm':
                gt['segmentation'] = to_rle(gt['segmentation'])
            gt['ignore'] = gt['ignore'] if 'ignore' in gt else 0
            gt['ignore'] = 'iscrowd' in gt and gt['iscrowd']
            self._gts[gt['image_id'], gt['category_id']].append(gt)
        for dt in self.dts_all:
            self._dts[dt['image_id'], dt['category_id']].append(dt)

    def evaluate(self):
        self._prepare()
        self.ious = {(imgId, catId): self.computeIoU(imgId, catId) for imgId in self.imgIds for catId in self.catIds}
        maxDet = MAX_DETS[-1]
        self.evalImgs = [self.evaluateImg(imgId, catId, areaRng, maxDet)
                         for catId in self.catIds for areaRng in AREA_RNG for imgId in self.imgIds]

    def computeIoU(self, imgId, catId):
        gt = self._gts[imgId, catId]
        dt = self._dts[imgId, catId]
        if len(gt) == 0 and len(dt) == 0:
            return []
        inds = np.argsort([-d['score'] for d in dt], kind='mergesort')
        dt = [dt[i] for i in inds]
        if len(dt) > MAX_DETS[-1]:
            dt = dt[0:MAX_DETS[-1]]
        if self.iouType == 'segm':
            g = [g['segmentation'] for g in gt]
            d = [d['segmentation'] for d in dt]
        else:
            g = [g['bbox'] for g in gt]
            d = [d['bbox'] for d in dt]
        iscrowd = [int(o['iscrowd']) for o in gt]
        if len(d) == 0 or len(g) == 0:
            return []
        return rle_iou(d, g, iscrowd) if self.iouType == 'segm' else bb_iou(d, g, iscrowd)

    def evaluateImg(self, imgId, catId, aRng, maxDet):
        gt = self._gts[imgId, catId]
        dt = self._dts[imgId, catId]
        if len(gt) == 0 and len(dt) == 0:
            return None
        for g in gt:
            if g['ignore'] or (g['area'] < aRng[0] or g['area'] > aRng[1]):
                g['_ignore'] = 1
            else:
                g['_ignore'] = 0
        gtind = np.argsort([g['_ignore'] for g in gt], kind='mergesort')
        gt = [gt[i] for i in gtind]
        dtind = np.argsort([-d['score'] for d in dt], kind='mergesort')
        dt = [dt[i] for i in dtind[0:maxDet]]
        iscrowd = [int(o['iscrowd']) for o in gt]
        ious = self.ious[imgId, catId][:, gtind] if len(self.ious[imgId, catId]) > 0 else self.ious[imgId, catId]
        T = len(IOU_THRS)
        G = len(gt)
        D = len(dt)
        gtm = np.zeros((T, G))
        dtm = np.zeros((T, D))
        gtIg = np.array([g['_ignore'] for g in gt])
        dtIg = np.zeros((T, D))
        if not len(ious) == 0:
            for tind, t in enumerate(IOU_THRS):
                for dind, d in enumerate(dt):
                    iou = min([t, 1 - 1e-10])
                    m = -1
                    for gind, g in enumerate(gt):
                        if gtm[tind, gind] > 0 and not iscrowd[gind]:
                            continue
                        if m > -1 and gtIg[m] == 0 and gtIg[gind] == 1:
                            break
                        if ious[dind, gind] < iou:
                            continue
                        iou = ious[dind, gind]
                        m = gind
                    if m == -1:
                        continue
                    dtIg[tind, dind] = gtIg[m]
                    dtm[tind, dind] = gt[m]['id']
                    gtm[tind, m] = d['id']
        a = np.array([d['area'] < aRng[0] or d['area'] > aRng[1] for d in dt]).reshape((1, len(dt)))
        dtIg = np.logical_or(dtIg, np.logical_and(dtm == 0, np.repeat(a, T, 0)))
        return {'image_id': imgId, 'category_id': catId, 'aRng': aRng, 'maxDet': maxDet,
                'dtIds': [d['id'] for d in dt], 'gtIds': [g['id'] for g in gt], 'dtMatches': dtm, 'gtMatches': gtm,
                'dtScores': [d['score'] for d in dt], 'gtIgnore': gtIg, 'dtIgnore': dtIg}

    def accumulate(self):
        T, R, K, A, M = len(IOU_THRS), len(REC_THRS), len(self.catIds), len(AREA_RNG), len(MAX_DETS)
        precision = -np.ones((T, R, K, A, M))
        recall = -np.ones((T, K, A, M))
        scores = -np.ones((T, R, K, A, M))
        I0, A0 = len(self.imgIds), len(AREA_RNG)
        for k in range(K):
            Nk = k * A0 * I0
            for a in range(A):
                Na = a * I0
                for m, maxDet in enumerate(MAX_DETS):
                    E = [self.evalImgs[Nk + Na + i] for i in range(I0)]
                    E = [e for e in E if e is not None]
                    if len(E) == 0:
                        continue
                    dtScores = np.concatenate([e['dtScores'][0:maxDet] for e in E])
                    inds = np.argsort(-dtScores, kind='mergesort')
                    dtScoresSorted = dtScores[inds]
                    dtm = np.concatenate([e['dtMatches'][:, 0:maxDet] for e in E], axis=1)[:, inds]
                    dtIg = np.concatenate([e['dtIgnore'][:, 0:maxDet] for e in E], axis=1)[:, inds]
                    gtIg = np.concatenate([e['gtIgnore'] for e in E])
                    npig = np.count_nonzero(gtIg == 0)
                    if npig == 0:
                        continue
                    tps = np.logical_and(dtm, np.logical_not(dtIg))
                    fps = np.logical_and(np.logical_not(dtm), np.logical_not(dtIg))
                    tp_sum = np.cumsum(tps, axis=1).astype(dtype=np.float64)
                    fp_sum = np.cumsum(fps, axis=1).astype(dtype=np.float64)
                    for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                        tp = np.array(tp)
                        fp = np.array(fp)
                        nd = len(tp)
                        rc = tp / npig
                        pr = tp / (fp + tp + np.spacing(1))
                        q = np.zeros((R,))
                        ss = np.zeros((R,))
                        recall[t, k, a, m] = rc[-1] if nd else 0
                        pr = pr.tolist()
                        q = q.tolist()
                        for i in range(nd - 1, 0, -1):
                            if pr[i] > pr[i - 1]:
                                pr[i - 1] = pr[i]
                        inds = np.searchsorted(rc, REC_THRS, side='left')
                        try:
                            for ri, pi in enumerate(inds):
                                q[ri] = pr[pi]
                                ss[ri] = dtScoresSorted[pi]
                        except IndexError:
                            pass
                        precision[t, :, k, a, m] = np.array(q)
                        scores[t, :, k, a, m] = np.array(ss)
        self.eval = {'precision': precision, 'recall': recall, 'scores': scores}

    def summarize(self):
        def _summarize(ap=1, iouThr=None, areaRng='all', maxDets=100):
            aind = [i for i, aRng in enumerate(AREA_LBL) if aRng == areaRng]
            mind = [i for i, mDet in enumerate(MAX_DETS) if mDet == maxDets]
            if ap == 1:
                s = self.eval['precision']
                if iouThr is not None:
                    s = s[np.where(iouThr == IOU_THRS)[0]]
                s = s[:, :, :, aind, mind]
            else:
                s = self.eval['recall']
                if iouThr is not None:
                    s = s[np.where(iouThr == IOU_THRS)[0]]
                s = s[:, :, aind, mind]
            return -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
        stats = np.zeros((12,))
        stats[0] = _summarize(1)
        stats[1] = _summarize(1, iouThr=.5, maxDets=MAX_DETS[2])
        stats[2] = _summarize(1, iouThr=.75, maxDets=MAX_DETS[2])
        stats[3] = _summarize(1, areaRng='small', maxDets=MAX_DETS[2])
        stats[4] = _summarize(1, areaRng='medium', maxDets=MAX_DETS[2])
        stats[5] = _summarize(1, areaRng='large', maxDets=MAX_DETS[2])
        stats[6] = _summarize(0, maxDets=MAX_DETS[0])
        stats[7] = _summarize(0, maxDets=MAX_DETS[1])
        stats[8] = _summarize(0, maxDets=MAX_DETS[2])
        stats[9] = _summarize(0, areaRng='small', maxDets=MAX_DETS[2])
        stats[10] = _summarize(0, areaRng='medium', maxDets=MAX_DETS[2])
        stats[11] = _summarize(0, areaRng='large', maxDets=MAX_DETS[2])
        self.stats = stats
        return stats


def format_results(images, cat_ids, iou_type):
    """The results list evaluate_boxes / evaluate_masks write, from per-image detections in im_post order:
    images = [(image_id, boxes fp32 [n,4], scores fp32 [n], cls int [n], segms list of RLE dicts or None)], cat_ids in
    class order (class j -> cat_ids[j - 1]).  Class-major, then ascending image id, then detection order; boxes go through
    dets.astype(float) and xyxy_to_xywh (w = x2 - x1 + 1 in float64)."""
    results = []
    order = sorted(range(len(images)), key=lambda i: images[i][0])
    for j, cat_id in enumerate(cat_ids, start=1):
        for i in order:
            image_id, boxes, scores, cls, segms = images[i]
            sel = np.flatnonzero(np.asarray(cls) == j)
            dets = np.hstack([np.asarray(boxes, np.float32)[sel], np.asarray(scores, np.float32)[sel, None]]).astype(np.float64)
            xy = dets[:, 0:2]
            wh = dets[:, 2:4] - dets[:, 0:2] + 1
            for r, d in enumerate(sel):
                res = {'image_id': image_id, 'category_id': cat_id, 'score': dets[r, 4]}
                if iou_type == 'bbox':
                    res['bbox'] = [xy[r, 0], xy[r, 1], wh[r, 0], wh[r, 1]]
                else:
                    res['segmentation'] = segms[d]
                results.append(res)
    return results


def evaluate(gt_anns, images, cat_ids, iou_type):
    """The whole evaluation: gt_anns with image_id; images as format_results takes them.  Returns the COCOeval object
    after evaluate / accumulate / summarize."""
    gts = [dict(a, id=a.get('id', i + 1)) for i, a in enumerate(gt_anns)]
    E = COCOeval(gts, load_res(format_results(images, cat_ids, iou_type), iou_type), [im[0] for im in images], cat_ids,
                 iou_type)
    E.evaluate()
    E.accumulate()
    E.summarize()
    return E
