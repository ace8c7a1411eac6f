"""Panoptic quality (PQ / SQ / RQ) and semantic-segmentation IoU evaluation on the device.

The reference evaluates on the host (dataset/base_dataset.py:209-330 evaluate_panoptic): `_converter_2ch_single_core`
turns every 2-channel prediction into segments, `_pq_compute_single_core` counts the (ground truth, prediction)
intersections and matches them, and `PQStat.pq_average` turns the per-category sums into the metrics.
`PanopticQuality` keeps the per-category sums (tp, fp, fn as int64, the IoU sum as fp64) on the device and adds one
image per `update()` with the kernels of csrc/pq.cu; only `pq_stat()` / `summarize()` copy them back.

    pq = PanopticQuality(gt_json["categories"])
    for ann, pan_2ch in zip(gt_json["annotations"], predictions):      # pan_2ch: uint8 [H,W,3] from unified_pan_result
        pq.update(pan_2ch, gt_png_rgb, ann["segments_info"])
    results = pq.summarize()                                            # {'All', 'Things', 'Stuff', 'per_class'}

The semantics are those of the reference, quirks included: stuff segments with different instance numbers merge, the
ground truth's `area` field (not its pixel count) enters the union, only the last crowd segment of a category counts,
ids in the PNG that are missing from `segments_info` take part in nothing, and a later duplicate id wins.

`SegmentationIoU` does the same for the semantic-segmentation mIoU of the reference's `evaluate_ssegs`
(dataset/cityscapes.py:445-514, coco.py:225-293, base_dataset.py:806-824 get_confusion_matrix).  The [C, C] confusion
matrix stays on the device as int64 and grows by one image per `update()` (csrc/sseg.cu); only `confusion_matrix()` /
`summarize()` copy it back.

    miou = SegmentationIoU(19)
    for pred, seg_gt in zip(fcn_outputs, gt_pngs):          # pred: int64 / uint8 label map; seg_gt: uint8 trainId PNG
        miou.update(pred, seg_gt)                           # or update(network_map, seg_gt, im_info) before the restore
    results = miou.summarize()                              # {'meanIU', 'IU_array', 'confusion_matrix'}

The reference's quirks are kept: prediction values wrap mod 256 (np.uint8), the prediction is resized to the ground truth
with Pillow's NEAREST rule (not cv2's), only gt == 255 is ignored, and a pixel counts in bin gt * C + pred only when
that bin exists, so gt rows >= C are dropped and predictions >= C alias into later rows.

`DetectionAP` computes the COCO box or mask AP of the reference's evaluate_boxes / evaluate_masks (pycocotools COCOeval
with its default Params) without the results JSON: update() matches one image on the device (csrc/cocoeval.cu), reading
the masks from im_post_rle's run lengths, and summarize() accumulates every image's records on the device and copies
precision / recall / scores back once.
"""
import collections
import ctypes as C

import numpy as np
import torch

from ._lib import UpsnetError, check, lib, ptr, stream_ptr
from .operators import label_restore_geometry, label_restore_index

MAX_GT = 4096          # UPSNET_PQ_MAX_GT: ground-truth segments per image
MAX_PAIRS = 65536      # UPSNET_PQ_MAX_PAIRS: distinct (ground truth, prediction) segment pairs per image
MAX_PRED = 2048        # UPSNET_PQ_MAX_PRED: prediction segments per image

_ERRORS = ((2, "more than %d ground-truth segments in one image" % MAX_GT),
           (4, "more than %d distinct (ground truth, prediction) segment pairs in one image" % MAX_PAIRS),
           (8, "invalid ground-truth table (ids must be unique in [1, 2^24), category ids in [0, 255))"),
           (16, "more than %d prediction segments in one image" % MAX_PRED),
           (32, "more than %d matches in one image (segments_info areas smaller than the segments)" % MAX_GT))


def pq_average(stat, categories, isthing):
    """PQStat.pq_average (base_dataset.py:73-97) on {category: (iou, tp, fp, fn)}; same arithmetic, same
    ZeroDivisionError when no category of the group has a segment."""
    pq, sq, rq, n = 0, 0, 0, 0
    per_class_results = {}
    for label, label_info in categories.items():
        if isthing is not None:
            cat_isthing = label_info['isthing'] == 1
            if isthing != cat_isthing:
                continue
        iou, tp, fp, fn = stat.get(label, (0.0, 0, 0, 0))
        if tp + fp + fn == 0:
            per_class_results[label] = {'pq': 0.0, 'sq': 0.0, 'rq': 0.0}
            continue
        n += 1
        pq_class = iou / (tp + 0.5 * fp + 0.5 * fn)
        sq_class = iou / tp if tp != 0 else 0
        rq_class = tp / (tp + 0.5 * fp + 0.5 * fn)
        per_class_results[label] = {'pq': pq_class, 'sq': sq_class, 'rq': rq_class, 'iou': iou, 'tp': tp, 'fp': fp, 'fn': fn}
        pq += pq_class
        sq += sq_class
        rq += rq_class
    return {'pq': pq / n, 'sq': sq / n, 'rq': rq / n, 'n': n}, per_class_results


def pack_segments(segments_info):
    """The ground-truth segment list -> int64 [5, G] (id, category_id, iscrowd, area, order), sorted by id.  Duplicate
    ids resolve like the reference's dict (base_dataset.py:525): the later entry wins, the first position is kept."""
    segs = {int(el['id']): el for el in segments_info}
    table = np.empty((5, len(segs)), np.int64)
    for i, (sid, el) in enumerate(segs.items()):
        table[:, i] = (sid, int(el['category_id']), int(el['iscrowd']), int(el['area']), i)
    return table[:, np.argsort(table[0], kind="stable")]


class PanopticQuality:
    """Per-category PQ accumulator on one CUDA device.  `categories`: the gt json's categories, as the dict
    {id: {'isthing': 0|1, ...}} the reference builds (a list of category dicts is accepted too).  Category ids must
    lie in [0, 255); class 255 of a prediction is void.  Calls on one object must be issued on one stream."""

    STAGING_SLOTS = 8

    def __init__(self, categories, device=None):
        if not isinstance(categories, dict):
            categories = {el['id']: el for el in categories}
        self.categories = categories
        flags = np.zeros(256, np.uint8)
        for cid, info in categories.items():
            if not 0 <= int(cid) < 255:
                raise ValueError("category id %r outside [0, 255)" % (cid,))
            flags[int(cid)] = 1 | (2 if info['isthing'] else 0)     # IdGenerator.get_color tests isthing for truth
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        assert self.device.type == "cuda", "PanopticQuality runs on a CUDA device (no CPU fallback)"
        self._flags = torch.from_numpy(flags).to(self.device)
        self._counts = torch.zeros((3, 256), dtype=torch.int64, device=self.device)    # tp, fp, fn
        self._iou = torch.zeros((256,), dtype=torch.float64, device=self.device)
        self._err = torch.zeros((1,), dtype=torch.int32, device=self.device)
        nb = C.c_size_t(0)
        check(lib().upsnet_pq_workspace_bytes(C.byref(nb)), "pq_workspace_bytes")
        self._ws = torch.empty((nb.value,), dtype=torch.uint8, device=self.device)
        # segment-table staging: a ring of pinned host / device buffer pairs, each guarded by the event of its last
        # H2D copy.  A slot used inside a CUDA-graph capture is taken out of the ring: the graph reads it at replay.
        self._stage = [(torch.empty((5 * MAX_GT,), dtype=torch.int64, pin_memory=True),
                        torch.empty((5 * MAX_GT,), dtype=torch.int64, device=self.device), None) for _ in range(self.STAGING_SLOTS)]
        self._next = 0
        self._captured = []

    def _image(self, x, name):
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(np.ascontiguousarray(x))
        if x.dtype != torch.uint8 or x.dim() != 3 or x.shape[2] != 3:
            raise ValueError("%s must be uint8 [H,W,3], got %s %s" % (name, x.dtype, tuple(x.shape)))
        return x.to(self.device, non_blocking=True).contiguous()

    def update(self, pan_2ch, gt_rgb, segments_info, check_errors=False):
        """Adds one image.  pan_2ch uint8 [H,W,3] (class, instance, -) as unified_pan_result writes it; gt_rgb the
        panoptic ground-truth PNG as decoded, uint8 RGB [H,W,3]; segments_info the image's gt json list.  Host tensors
        are copied to the device once; the segment table goes through a pinned staging buffer.  Nothing waits for the
        device unless check_errors=True, which raises at once on an error flag (one int copied back)."""
        pan, gt = self._image(pan_2ch, "pan_2ch"), self._image(gt_rgb, "gt_rgb")
        if pan.shape != gt.shape:
            raise ValueError("pan_2ch %s and gt_rgb %s differ in size" % (tuple(pan.shape), tuple(gt.shape)))
        H, W = int(pan.shape[0]), int(pan.shape[1])
        table = pack_segments(segments_info)
        G = table.shape[1]
        capturing = torch.cuda.is_current_stream_capturing()
        if not self._stage:
            raise UpsnetError("PanopticQuality: every staging slot is held by a captured CUDA graph")
        k = self._next % len(self._stage)
        host, tdev, ev = self._stage[k]
        if 0 < G <= MAX_GT:             # a larger table is only counted: the device raises the error flag without reading it
            if ev is not None and not capturing:
                ev.synchronize()        # the H2D copy that last read this pinned slot (STAGING_SLOTS updates ago)
            # (torch.cuda.graph synchronises the device before a capture starts, so no copy is pending then)
            host[:5 * G].numpy()[...] = table.reshape(-1)
            tdev[:5 * G].copy_(host[:5 * G], non_blocking=True)
        if capturing:
            self._captured.append(self._stage.pop(k))
        else:
            if 0 < G <= MAX_GT:
                ev = torch.cuda.Event()
                ev.record(torch.cuda.current_stream(self.device))
                self._stage[k] = (host, tdev, ev)
            self._next += 1
        with torch.cuda.device(self.device):
            check(lib().upsnet_pq_update(ptr(pan), ptr(gt), H, W, ptr(tdev), G, ptr(self._flags), ptr(self._counts),
                                         ptr(self._iou), ptr(self._err), ptr(self._ws), self._ws.numel(),
                                         stream_ptr(self.device)), "pq_update")
        if check_errors:
            self.check_errors()

    def check_errors(self):
        """Raises if any update() so far hit an error (the flags are sticky until reset())."""
        e = int(self._err.item())
        if e & 1:
            raise KeyError("a prediction segment has a category id that is not in the categories (base_dataset.py:538)")
        for bit, msg in _ERRORS:
            if e & bit:
                raise UpsnetError("pq_update: " + msg)

    def pq_stat(self):
        """{category id: {'iou', 'tp', 'fp', 'fn'}} for every category with a segment so far (PQStat.pq_per_cat;
        categories outside the category table are kept, as the reference's defaultdict does)."""
        counts = self._counts.cpu().numpy()
        iou = self._iou.cpu().numpy()
        out = {}
        for c in np.flatnonzero(counts.any(0) | (iou != 0)):
            out[int(c)] = {'iou': float(iou[c]), 'tp': int(counts[0, c]), 'fp': int(counts[1, c]), 'fn': int(counts[2, c])}
        return out

    def summarize(self):
        """What the reference's pq_compute returns: {'All', 'Things', 'Stuff'} each {'pq','sq','rq','n'}, and
        'per_class' (base_dataset.py:290-298)."""
        self.check_errors()
        stat = {c: (v['iou'], v['tp'], v['fp'], v['fn']) for c, v in self.pq_stat().items()}
        results = {}
        for name, isthing in (("All", None), ("Things", True), ("Stuff", False)):
            results[name], per_class_results = pq_average(stat, self.categories, isthing)
            if name == 'All':
                results['per_class'] = per_class_results
        return results

    def reset(self):
        self._counts.zero_()
        self._iou.zero_()
        self._err.zero_()


MAX_SSEG_CLASSES = 224     # UPSNET_SSEG_MAX_CLASSES: a C*C uint32 histogram per block fits in shared memory


def pil_nearest_index(n_in, n_out):
    """Source indices of PIL's Image.resize(..., Image.NEAREST) along one axis (ImagingScaleAffine): with a = n_in / n_out,
    output i reads int(acc_i), acc_0 = a / 2 and acc_{i+1} = acc_i + a summed one after the other in double.  This is
    neither cv2's rule nor floor((i + 0.5) * a); equal sizes give the identity."""
    a = n_in / n_out
    idx = np.add.accumulate(np.r_[a * 0.5, np.full(n_out - 1, a)]).astype(np.int64)       # sequential, then truncated
    assert idx[0] >= 0 and idx[-1] < n_in
    return idx


def sseg_index_tables(pred_hw, gt_hw, im_info=None):
    """int32 (row_src [H], col_src [W]) for upsnet_sseg_update.  Without im_info the prediction is resized from pred_hw to
    the ground-truth size gt_hw by Pillow's rule.  With im_info the prediction is the network-resolution map (padded
    [Hp, Wp]); the tables then compose the test script's crop + cv2 restore (label_restore, upsnet_end2end_test.py:259-266)
    with Pillow's resize from the restored size to gt_hw, so they pick the pixels the reference's loop would."""
    (ph, pw), (H, W) = (int(v) for v in pred_hw), (int(v) for v in gt_hw)
    if im_info is None:
        rows, cols = pil_nearest_index(ph, H), pil_nearest_index(pw, W)
    else:
        h, w, fx, oh, ow = label_restore_geometry(im_info)
        if not (0 < h <= ph and 0 < w <= pw):
            raise ValueError("im_info crop (%d, %d) outside the %dx%d label map" % (h, w, ph, pw))
        if oh <= 0 or ow <= 0:
            raise ValueError("im_info restores the map to an empty %dx%d image" % (oh, ow))
        rows = label_restore_index(oh, fx, h)[pil_nearest_index(oh, H)]
        cols = label_restore_index(ow, fx, w)[pil_nearest_index(ow, W)]
    return rows.astype(np.int32), cols.astype(np.int32)


class SegmentationIoU:
    """Semantic-segmentation confusion matrix and mIoU of the reference's evaluate_ssegs, accumulated on one CUDA device.
    1 <= num_classes <= 224 (19 for Cityscapes, 133 for COCO).  Calls on one object must be issued on one stream."""

    TABLE_CACHE = 16       # index-table geometries kept on the device (LRU)

    def __init__(self, num_classes, device=None):
        if not 1 <= int(num_classes) <= MAX_SSEG_CLASSES:
            raise ValueError("num_classes %r outside [1, %d]" % (num_classes, MAX_SSEG_CLASSES))
        self.num_classes = int(num_classes)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        assert self.device.type == "cuda", "SegmentationIoU runs on a CUDA device (no CPU fallback)"
        self._acc = torch.zeros((self.num_classes ** 2,), dtype=torch.int64, device=self.device)
        self._tables = collections.OrderedDict()
        self._captured = []    # tables a captured CUDA graph reads at replay: never freed by the LRU

    def _map(self, x, name, dtypes, max_dim):
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(np.ascontiguousarray(x))
        if x.dtype not in dtypes or not 2 <= x.dim() <= max_dim or any(int(s) != 1 for s in x.shape[:-2]):
            raise ValueError("%s must be %s [h,w]%s, got %s %s"
                             % (name, "/".join(str(d).replace("torch.", "") for d in dtypes),
                                " / [1,h,w] / [1,1,h,w]" if max_dim > 2 else "", x.dtype, tuple(x.shape)))
        if x.numel() == 0:
            raise ValueError("%s is empty: %s" % (name, tuple(x.shape)))
        return x.reshape(x.shape[-2:]).to(self.device, non_blocking=True).contiguous()

    def _index_tables(self, pred_hw, gt_hw, im_info):
        info = None if im_info is None else tuple(np.asarray(im_info, np.float32).reshape(-1)[:3].tolist())
        key = (pred_hw, gt_hw, info)
        tab = self._tables.get(key)
        if tab is not None:
            self._tables.move_to_end(key)
            return tab
        if torch.cuda.is_current_stream_capturing():
            raise UpsnetError("SegmentationIoU: new geometry %s inside a CUDA-graph capture; call update() once outside "
                              "the capture" % (key,))
        rows, cols = sseg_index_tables(pred_hw, gt_hw, im_info)
        host = torch.from_numpy(np.concatenate([rows, cols])).pin_memory()
        tab = host.to(self.device, non_blocking=True)
        self._tables[key] = tab
        while len(self._tables) > self.TABLE_CACHE:
            self._tables.popitem(last=False)
        return tab

    def update(self, pred, seg_gt, im_info=None):
        """Adds one image.  pred int64 or uint8 [h,w] / [1,h,w] / [1,1,h,w]: the semantic label map at any size (it is
        resized to seg_gt by Pillow's rule), or with im_info ([h, w, scale] as the data loader gives it) the
        network-resolution map before the restore.  seg_gt uint8 [H,W], the trainId PNG as decoded.  Host arrays are
        copied to the device once; nothing waits for the device."""
        p = self._map(pred, "pred", (torch.int64, torch.uint8), 4)
        g = self._map(seg_gt, "seg_gt", (torch.uint8,), 2)
        pred_hw, gt_hw = tuple(int(s) for s in p.shape), tuple(int(s) for s in g.shape)
        tab = self._index_tables(pred_hw, gt_hw, im_info)
        if torch.cuda.is_current_stream_capturing():
            self._captured.append(tab)
        H, W = gt_hw
        with torch.cuda.device(self.device):
            check(lib().upsnet_sseg_update(ptr(p), p.element_size(), pred_hw[1], ptr(tab), C.c_void_p(tab.data_ptr() + 4 * H),
                                           ptr(g), H, W, self.num_classes, ptr(self._acc), stream_ptr(self.device)),
                  "sseg_update")

    def confusion_matrix(self):
        """float64 [C, C] (row = ground truth, column = prediction): the matrix the reference accumulates."""
        C_ = self.num_classes
        return self._acc.cpu().numpy().reshape(C_, C_).astype(np.float64)

    def summarize(self):
        """evaluate_ssegs's evaluation_results: {'meanIU', 'IU_array', 'confusion_matrix'}, with its arithmetic (the mean
        runs over all C classes, so a class that never appears counts as 0)."""
        confusion_matrix = self.confusion_matrix()
        pos = confusion_matrix.sum(1)
        res = confusion_matrix.sum(0)
        tp = np.diag(confusion_matrix)
        IU_array = (tp / np.maximum(1.0, pos + res - tp))
        mean_IU = IU_array.mean()
        return {'meanIU': mean_IU, 'IU_array': IU_array, 'confusion_matrix': confusion_matrix}

    def reset(self):
        self._acc.zero_()


# ---------------------------------------------------------------------------------------------------------------------
# COCO box / mask AP: pycocotools COCOeval ('bbox' / 'segm', default Params) as the reference's evaluate_boxes
# (base_dataset.py:181-204) and evaluate_masks (coco.py:194-222) run it, on the device (csrc/cocoeval.cu).
# ---------------------------------------------------------------------------------------------------------------------
MAX_AP_DET = 2048          # UPSNET_COCOEVAL_MAX_DET: detections per update()
MAX_AP_GT = 1024           # UPSNET_COCOEVAL_MAX_GT: ground truths per image
MAX_AP_GT_CAT = 192        # UPSNET_COCOEVAL_MAX_GT_CAT: ground truths per (image, category)
MAX_AP_CATEGORIES = 256    # UPSNET_COCOEVAL_MAX_CATEGORIES
MAX_AP_IMAGES = 1 << 17    # UPSNET_COCOEVAL_MAX_IMAGES
IOU_THRS = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)    # COCOeval Params.setDetParams
MAX_DETS = [1, 10, 100]

_AP_ERRORS = ((1, "more than %d detections in one image" % MAX_AP_DET),
              (2, "more than %d ground truths in one image" % MAX_AP_GT),
              (4, "more than %d ground truths of one category in one image" % MAX_AP_GT_CAT),
              (8, "a detection class index outside [1, number of categories]"),
              (16, "more records than record_capacity (kept detections over all images)"),
              (32, "a mask RLE that does not cover the image (size mismatch, or im_post_rle's buffer overflowed)"))


def _mask_counts(mask):
    """maskApi.c rleEncode of a [H,W] mask: run lengths of the column-major flattening, starting with the zeros run."""
    v = (np.asarray(mask) != 0).astype(np.uint8).flatten(order="F")
    if v.size == 0:
        return np.zeros(0, np.uint32)
    edges = np.concatenate([[0], np.flatnonzero(v[1:] != v[:-1]) + 1, [v.size]])
    cnts = np.diff(edges)
    if v[0]:
        cnts = np.concatenate([[0], cnts])
    return cnts.astype(np.uint32)


def gt_rle(segmentation):
    """A ground-truth `segmentation` -> (h, w, uint32 run lengths).  Accepts a compressed or uncompressed COCO RLE dict or
    a [H,W] mask.  Polygons are rejected: rasterise them first (COCO.annToRLE(ann))."""
    from .operators import rle_from_string
    if isinstance(segmentation, dict):
        h, w = (int(v) for v in segmentation["size"])
        cnts = segmentation["counts"]
        counts = rle_from_string(cnts) if isinstance(cnts, (str, bytes)) else np.asarray(cnts, np.int64).astype(np.uint32)
        return h, w, counts
    if isinstance(segmentation, list):
        raise ValueError("polygon segmentations are not rasterised here: pass COCO.annToRLE(ann) as the segmentation")
    if isinstance(segmentation, torch.Tensor):
        segmentation = segmentation.cpu().numpy()
    m = np.asarray(segmentation)
    if m.ndim != 2:
        raise ValueError("a mask segmentation must be [H,W], got shape %s" % (m.shape,))
    return int(m.shape[0]), int(m.shape[1]), _mask_counts(m)


def summarize_stats(precision, recall):
    """COCOeval.summarize()'s 12 stats (_summarizeDets) from precision [T,R,K,A,M] and recall [T,K,A,M]."""
    area_lbl = ['all', 'small', 'medium', 'large']

    def _summarize(ap=1, iouThr=None, areaRng='all', maxDets=100):
        aind = [i for i, aRng in enumerate(area_lbl) if aRng == areaRng]
        mind = [i for i, mDet in enumerate(MAX_DETS) if mDet == maxDets]
        s = precision if ap == 1 else recall
        if iouThr is not None:
            s = s[np.where(iouThr == IOU_THRS)[0]]
        s = s[:, :, :, aind, mind] if ap == 1 else s[:, :, aind, mind]
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
    return stats


def per_class_ap(precision):
    """The AP values log_detection_eval_metrics (base_dataset.py:674-716) logs: for IoU [0.50, 0.95] and [0.50, 0.50], the
    mean over precision[lo:hi+1, :, :, 0, 2] > -1 and the same per K index (the reference slices class j at K index
    j - 1).  {'0.50:0.95': {'mean', 'per_class'}, '0.50:0.50': {...}}; an empty selection gives nan, as np.mean does."""
    def thr_ind(thr):
        return int(np.where((IOU_THRS > thr - 1e-5) & (IOU_THRS < thr + 1e-5))[0][0])

    def mean(p):
        sel = p[p > -1]
        return float(np.mean(sel)) if sel.size else float("nan")
    out = {}
    lo = thr_ind(0.5)
    for hi_thr in (0.95, 0.5):
        hi = thr_ind(hi_thr)
        p = precision[lo:hi + 1, :, :, 0, 2]
        out["0.50:%.2f" % hi_thr] = {"mean": mean(p), "per_class": [mean(p[:, :, k]) for k in range(p.shape[2])]}
    return out


class DetectionAP:
    """COCO box ('bbox') or mask ('segm') AP of the reference's evaluate_boxes / evaluate_masks, computed on one CUDA
    device.  `categories`: the gt json's category list (or {id: info}).  The K axis of the results is the category ids
    sorted (COCOeval's p.catIds); a detection of class j (JsonDataset order: the j-th category of `categories`, 1-based)
    counts for that category's id.  Every image of the dataset must be passed to update() once, with or without
    detections.  Calls on one object must be issued on one stream.

        ap = DetectionAP(gt_json["categories"], iou_type="segm")
        for image_id, anns, (boxes, scores, cls_inds, counts, run_len) in data:
            ap.update(image_id, anns, boxes, scores, cls_inds, rle=(counts, run_len))
        res = ap.summarize()            # {'stats', 'precision', 'recall', 'scores', 'per_class_ap'}
    """

    STAGING_SLOTS = 8

    def __init__(self, categories, iou_type="segm", device=None, record_capacity=1 << 20):
        if iou_type not in ("bbox", "segm"):
            raise ValueError("iou_type must be 'bbox' or 'segm', got %r" % (iou_type,))
        if isinstance(categories, dict):
            categories = [dict(v, id=k) for k, v in categories.items()]
        ids = [int(c["id"]) for c in categories]
        if not 1 <= len(ids) <= MAX_AP_CATEGORIES or len(set(ids)) != len(ids):
            raise ValueError("need 1 to %d distinct category ids, got %d (%d distinct)"
                             % (MAX_AP_CATEGORIES, len(ids), len(set(ids))))
        self.iou_type = iou_type
        self.cat_ids = sorted(ids)
        self._cat_to_k = {cid: k for k, cid in enumerate(self.cat_ids)}
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        assert self.device.type == "cuda", "DetectionAP runs on a CUDA device (no CPU fallback)"
        K = len(ids)
        self._cls_to_k = torch.tensor([-1] + [self._cat_to_k[c] for c in ids], dtype=torch.int32, device=self.device)
        self.record_capacity = int(record_capacity)
        self._records = torch.empty((self.record_capacity, 4), dtype=torch.int64, device=self.device)   # 32-byte records
        self._n_rec = torch.zeros((1,), dtype=torch.int32, device=self.device)
        self._npig = torch.zeros((K, 4), dtype=torch.int64, device=self.device)
        self._err = torch.zeros((1,), dtype=torch.int32, device=self.device)
        self._ws = torch.empty((0,), dtype=torch.uint8, device=self.device)
        self._stage = [[torch.empty((0,), dtype=torch.uint8), torch.empty((0,), dtype=torch.uint8, device=self.device), None]
                       for _ in range(self.STAGING_SLOTS)]
        self._next = 0
        self._image_ids = []
        self._seen = set()

    def _det(self, x, dtype, shape, name):
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(np.ascontiguousarray(x))
        x = torch.as_tensor(x)
        if tuple(x.shape) != shape:
            raise ValueError("%s must have shape %s, got %s" % (name, shape, tuple(x.shape)))
        return x.to(self.device, dtype, non_blocking=True).contiguous()

    def _gt_table(self, gt_anns):
        """fp64 [9][G] (K index, iscrowd, area, x, y, w, h, rle h, rle w) and, for segm, the run lengths and offsets."""
        G = len(gt_anns)
        table = np.zeros((9, G), np.float64)
        runs = []
        for j, ann in enumerate(gt_anns):
            cid = int(ann["category_id"])
            if cid not in self._cat_to_k:
                raise KeyError("ground-truth category_id %d is not in the categories" % cid)
            table[0, j] = self._cat_to_k[cid]
            table[1, j] = 1.0 if ann.get("iscrowd", 0) else 0.0        # _prepare: ignore = iscrowd
            table[2, j] = float(ann["area"])
            if self.iou_type == "bbox":
                table[3:7, j] = [float(v) for v in ann["bbox"]]
            else:
                h, w, cnts = gt_rle(ann["segmentation"])
                table[7, j], table[8, j] = h, w
                runs.append(cnts)
        offs = np.zeros(G + 1, np.int64)
        if runs:
            offs[1:] = np.cumsum([r.size for r in runs])
        counts = np.concatenate(runs).astype(np.uint32) if runs else np.zeros(0, np.uint32)
        return table, offs, counts

    def _stage_gt(self, table, offs, counts):
        """Copies the ground truths through a ring of pinned buffers; returns device pointers (table, offsets, counts)."""
        G = table.shape[1]
        nt, no = 8 * table.size, 8 * offs.size
        nbytes = nt + no + 4 * counts.size
        k = self._next % len(self._stage)
        self._next += 1
        host, dev, ev = self._stage[k]
        if ev is not None:
            ev.synchronize()           # the H2D copy that last read this pinned slot (STAGING_SLOTS updates ago)
        if host.numel() < nbytes:
            size = max(nbytes, 2 * host.numel(), 1 << 16)
            host = torch.empty((size,), dtype=torch.uint8, pin_memory=True)
            dev = torch.empty((size,), dtype=torch.uint8, device=self.device)
        h = host.numpy()
        h[:nt] = table.reshape(-1).view(np.uint8)
        h[nt:nt + no] = offs.view(np.uint8)
        h[nt + no:nbytes] = counts.view(np.uint8)
        if nbytes:
            dev[:nbytes].copy_(host[:nbytes], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        self._stage[k] = [host, dev, ev]
        base = dev.data_ptr()
        return (C.c_void_p(base), C.c_void_p(base + nt), C.c_void_p(base + nt + no)) if G else (None, None, None)

    def update(self, image_id, gt_anns, boxes, scores, cls_inds, rle=None, n_dev=None, im_size=None):
        """Adds one image: COCOeval.evaluate() for its detections and ground truths.
        gt_anns: the image's instance annotations (category_id, iscrowd, area, and bbox for 'bbox' / segmentation for
        'segm', as a compressed or uncompressed RLE or a [H,W] mask).  boxes fp32 [n,4] x1 y1 x2 y2, scores fp32 [n],
        cls_inds int64 [n] class indices in [1, K], in im_post order.  rle = (counts, run_len) as ops.im_post_rle returns
        them (segm only; they stay on the device).  n_dev: optional device int32 count, as for im_post_rle.  im_size:
        (H, W) of the detection masks, by default the ground truths' RLE size.  Nothing waits for the device."""
        if image_id in self._seen:
            raise ValueError("image id %r was already added" % (image_id,))
        if len(self._image_ids) >= MAX_AP_IMAGES:
            raise ValueError("more than %d images" % MAX_AP_IMAGES)
        n = int(boxes.shape[0]) if hasattr(boxes, "shape") else len(boxes)
        b = self._det(boxes, torch.float32, (n, 4), "boxes")
        s = self._det(scores, torch.float32, (n,), "scores")
        c = self._det(cls_inds, torch.int64, (n,), "cls_inds")
        segm = self.iou_type == "segm"
        if segm and rle is None:
            raise ValueError("iou_type 'segm' needs rle=(counts, run_len)")
        table, offs, counts = self._gt_table(gt_anns)
        G = table.shape[1]
        cnt, rl, cap, H, W = None, None, 0, 0, 0
        if segm:
            cnt, rl = rle[0], rle[1]
            if not (cnt.is_cuda and rl.is_cuda) or cnt.dim() != 2 or cnt.shape[0] < n or rl.numel() < n \
                    or cnt.element_size() != 4 or rl.dtype != torch.int32:
                raise ValueError("rle must be im_post_rle's device tensors (counts [n, cap] 32-bit, run_len int32 [n])")
            cnt, rl, cap = cnt.contiguous(), rl.contiguous(), int(cnt.shape[1])
            if im_size is not None:
                H, W = (int(v) for v in im_size)
            elif G:
                H, W = int(table[7, 0]), int(table[8, 0])
            nb = C.c_size_t(0)
            check(lib().upsnet_cocoeval_workspace_bytes(n, cap, int(counts.size), C.byref(nb)), "cocoeval_workspace_bytes")
            if self._ws.numel() < nb.value:
                self._ws = torch.empty((nb.value,), dtype=torch.uint8, device=self.device)
        if n_dev is not None and (not n_dev.is_cuda or n_dev.dtype != torch.int32):
            raise ValueError("n_dev must be a device int32 tensor")
        if G <= MAX_AP_GT:
            t_ptr, o_ptr, c_ptr = self._stage_gt(table, offs, counts)
        else:                          # only counted: the device raises the error flag without reading the table
            t_ptr = o_ptr = c_ptr = None
        slot = len(self._image_ids)
        with torch.cuda.device(self.device):
            check(lib().upsnet_cocoeval_image(int(segm), ptr(b), ptr(s), ptr(c), n, ptr(n_dev), ptr(cnt), cap, ptr(rl), H, W,
                                              t_ptr, G, c_ptr, o_ptr, len(self.cat_ids), ptr(self._cls_to_k), slot,
                                              ptr(self._records), self.record_capacity, ptr(self._n_rec), ptr(self._npig),
                                              ptr(self._err), ptr(self._ws), self._ws.numel(), stream_ptr(self.device)),
                  "cocoeval_image")
        self._image_ids.append(image_id)
        self._seen.add(image_id)

    def check_errors(self):
        """Raises if any update() so far hit an error (the flags are sticky until reset())."""
        e = int(self._err.item())
        for bit, msg in _AP_ERRORS:
            if e & bit:
                raise UpsnetError("cocoeval: " + msg)

    def accumulate(self):
        """COCOeval.accumulate(): {'precision' [10,101,K,4,3], 'recall' [10,K,4,3], 'scores' [10,101,K,4,3]} fp64 numpy."""
        self.check_errors()
        N = int(self._n_rec.item())
        K = len(self.cat_ids)
        rank = np.empty(len(self._image_ids), np.int32)
        rank[np.argsort(np.asarray(self._image_ids), kind="stable")] = np.arange(len(self._image_ids), dtype=np.int32)
        rank_d = torch.from_numpy(rank).to(self.device)
        nb = C.c_size_t(0)
        check(lib().upsnet_cocoeval_accumulate_workspace_bytes(N, C.byref(nb)), "cocoeval_accumulate_workspace_bytes")
        ws = torch.empty((max(nb.value, 1),), dtype=torch.uint8, device=self.device)
        f64 = dict(dtype=torch.float64, device=self.device)
        out = torch.empty((2 * 10 * 101 * K * 12 + 10 * K * 12,), **f64)
        precision = out[:10 * 101 * K * 12].view(10, 101, K, 4, 3)
        scores = out[10 * 101 * K * 12:2 * 10 * 101 * K * 12].view(10, 101, K, 4, 3)
        recall = out[2 * 10 * 101 * K * 12:].view(10, K, 4, 3)
        with torch.cuda.device(self.device):
            check(lib().upsnet_cocoeval_accumulate(ptr(self._records), N, ptr(rank_d), ptr(self._npig), K, ptr(precision),
                                                   ptr(recall), ptr(scores), ptr(ws), ws.numel(), stream_ptr(self.device)),
                  "cocoeval_accumulate")
        host = out.cpu().numpy()                                         # the one copy back
        n1 = 10 * 101 * K * 12
        return {"precision": host[:n1].reshape(10, 101, K, 4, 3), "scores": host[n1:2 * n1].reshape(10, 101, K, 4, 3),
                "recall": host[2 * n1:].reshape(10, K, 4, 3)}

    def summarize(self):
        """{'stats': COCOeval.stats (12 floats), 'precision', 'recall', 'scores', 'per_class_ap'} (per_class_ap: the values
        log_detection_eval_metrics logs, see per_class_ap())."""
        ev = self.accumulate()
        return {"stats": summarize_stats(ev["precision"], ev["recall"]), "precision": ev["precision"],
                "recall": ev["recall"], "scores": ev["scores"], "per_class_ap": per_class_ap(ev["precision"])}

    def reset(self):
        self._n_rec.zero_()
        self._npig.zero_()
        self._err.zero_()
        self._image_ids = []
        self._seen = set()
