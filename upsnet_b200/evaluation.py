"""Panoptic quality (PQ / SQ / RQ) evaluation on the device.

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
"""
import ctypes as C

import numpy as np
import torch

from ._lib import UpsnetError, check, lib, ptr, stream_ptr

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
