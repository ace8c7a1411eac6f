"""Device-resident restatement of the reference's CPU detection glue that sits between the hot
kernels (SURVEY.md section 8 rows a6, a10; F8: >=6 host round trips per image in the reference).

  generate_anchors / level anchors      rpn/generate_anchors.py:50-76,156-206;
                                        operators/functions/pyramid_proposal.py:73-100
  bbox_transform / clip_boxes           bbox/bbox_transform.py:290-330, :45-60
  pyramid_proposals                     operators/functions/pyramid_proposal.py:41-222 +
                                        operators/modules/pyramid_proposal.py:36-67
  mask_roi                              operators/modules/mask_roi.py:36-146

Tensors stay on the GPU; NMS is the segmented device kernel (one launch for all levels / classes).
The remaining host synchronisations are size reads (counts), noted inline.
"""
import math

import numpy as np
import torch

from . import operators as _ops
from .operators import nms_segmented

FUSED = {"on": True}   # CUDA tensors: fused decode / MaskROI kernels (detection.cu); False = torch restatement

BBOX_XFORM_CLIP = math.log(1000. / 16.)


def generate_anchors(stride, sizes, aspect_ratios=(0.5, 1, 2)):
    """Anchors (x1,y1,x2,y2) centred on (stride-1)/2: ratio enumeration with np.round on the
    widths/heights of the base window, then scale enumeration (float64, like the reference)."""
    scales = np.array(sizes, dtype=np.float64) / stride
    ratios = np.array(aspect_ratios, dtype=np.float64)
    base = float(stride)
    ctr = 0.5 * (base - 1)
    area = base * base
    ws = np.round(np.sqrt(area / ratios))
    hs = np.round(ws * ratios)
    out = []
    for w, h in zip(ws, hs):
        for s in scales:
            W, H = w * s, h * s
            out.append([ctr - 0.5 * (W - 1), ctr - 0.5 * (H - 1), ctr + 0.5 * (W - 1), ctr + 0.5 * (H - 1)])
    return np.array(out, dtype=np.float64)


def level_anchors(stride, height, width, scales=(8,), ratios=(0.5, 1, 2)):
    """All shifted anchors of one level, rows ordered (h, w, a) (pyramid_proposal.py:83-100),
    cast to float32 as bbox_transform does (bbox_transform.py:298)."""
    sub = generate_anchors(stride, np.array(scales) * stride, ratios)
    sx, sy = np.meshgrid(np.arange(0, width) * stride, np.arange(0, height) * stride)
    shifts = np.vstack((sx.ravel(), sy.ravel(), sx.ravel(), sy.ravel())).transpose()
    A, K = sub.shape[0], shifts.shape[0]
    anchors = sub.reshape((1, A, 4)) + shifts.reshape((1, K, 4)).transpose((1, 0, 2))
    return anchors.reshape((K * A, 4)).astype(np.float32)


def bbox_transform(boxes, deltas, weights=(1., 1., 1., 1.)):
    """boxes [N,4], deltas [N,4K] -> [N,4K] (float32 arithmetic, same operation order)."""
    widths = boxes[:, 2] - boxes[:, 0] + 1.0
    heights = boxes[:, 3] - boxes[:, 1] + 1.0
    ctr_x = boxes[:, 0] + 0.5 * widths
    ctr_y = boxes[:, 1] + 0.5 * heights
    wx, wy, ww, wh = weights
    dx = deltas[:, 0::4] / wx
    dy = deltas[:, 1::4] / wy
    dw = torch.clamp(deltas[:, 2::4] / ww, max=BBOX_XFORM_CLIP)
    dh = torch.clamp(deltas[:, 3::4] / wh, max=BBOX_XFORM_CLIP)
    pcx = dx * widths[:, None] + ctr_x[:, None]
    pcy = dy * heights[:, None] + ctr_y[:, None]
    pw = torch.exp(dw) * widths[:, None]
    ph = torch.exp(dh) * heights[:, None]
    out = torch.empty_like(deltas)
    out[:, 0::4] = pcx - 0.5 * pw
    out[:, 1::4] = pcy - 0.5 * ph
    out[:, 2::4] = pcx + 0.5 * pw - 1
    out[:, 3::4] = pcy + 0.5 * ph - 1
    return out


def clip_boxes(boxes, im_h, im_w):
    """im_h, im_w: Python floats, or 0-dim tensors on the boxes' device (the bounds are then read when the clamp runs, so
    the clip is the same inside a captured graph for every image size written to the row they come from)."""
    if torch.is_tensor(im_w):
        # clamp_(min=0, max=tensor) would stage the scalar bound through host memory, which a capture does not allow
        for c, lim in ((0, im_w), (1, im_h), (2, im_w), (3, im_h)):
            boxes[:, c::4].clamp_min_(0).clamp_max_(lim - 1)
        return boxes
    boxes[:, 0::4].clamp_(min=0, max=im_w - 1)
    boxes[:, 1::4].clamp_(min=0, max=im_h - 1)
    boxes[:, 2::4].clamp_(min=0, max=im_w - 1)
    boxes[:, 3::4].clamp_(min=0, max=im_h - 1)
    return boxes


class ProposalGenerator:
    """PyramidProposal (individual_proposals=True, the shipped setting: config.py:123)."""

    def __init__(self, feat_stride=(4, 8, 16, 32, 64), scales=(8,), ratios=(0.5, 1, 2), pre_nms_top_n=1000,
                 post_nms_top_n=1000, nms_thresh=0.7, min_size=0):
        self.feat_stride, self.scales, self.ratios = feat_stride, scales, ratios
        self.pre, self.post, self.thresh, self.min_size = pre_nms_top_n, post_nms_top_n, nms_thresh, min_size
        self._anchors = {}

    def anchors(self, lvl, h, w, device):
        key = (lvl, h, w, str(device))
        if key not in self._anchors:
            self._anchors[key] = torch.from_numpy(
                level_anchors(self.feat_stride[lvl], h, w, self.scales, self.ratios)).to(device)
        return self._anchors[key]

    def __call__(self, cls_probs, bbox_preds, im_info):
        """cls_probs[l] [1,A,h,w] (sigmoid), bbox_preds[l] [1,4A,h,w]; im_info (H, W, scale).
        Returns rois [R<=post,5] (batch 0), scores [R]."""
        dev = cls_probs[0].device
        im_h, im_w, im_scale = float(im_info[0]), float(im_info[1]), float(im_info[2])
        L = len(cls_probs)
        boxes_l, scores_l, lens = [], [], []
        for l in range(L):
            A = cls_probs[l].shape[1]
            h, w = cls_probs[l].shape[-2:]
            scores = cls_probs[l][0].permute(1, 2, 0).reshape(-1)                 # (h, w, a)
            deltas = bbox_preds[l][0].reshape(A, 4, h, w).permute(2, 3, 0, 1).reshape(-1, 4)
            k = min(self.pre, scores.numel()) if self.pre > 0 else scores.numel()
            top_s, top_i = torch.topk(scores, k, sorted=True)                     # descending
            props = bbox_transform(self.anchors(l, h, w, dev)[top_i], deltas[top_i])
            props = clip_boxes(props, im_h, im_w)
            if self.min_size > 0:  # config.test.rpn_min_size = 0 in every shipped yaml
                ws = props[:, 2] - props[:, 0] + 1
                hs = props[:, 3] - props[:, 1] + 1
                keep = (ws >= self.min_size * im_scale) & (hs >= self.min_size * im_scale)
                props, top_s = props[keep], top_s[keep]                           # host sync (size)
            boxes_l.append(props); scores_l.append(top_s); lens.append(props.shape[0])
        boxes = torch.cat(boxes_l)
        scores = torch.cat(scores_l)
        offs = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=dev)
        max_len = max(max(lens), 1)
        keep, cnt = nms_segmented(boxes, offs, max_len, self.thresh)             # one launch, all levels
        # gather kept boxes of every level without leaving the device
        pos = torch.arange(max_len, device=dev)[None, :]
        limit = cnt.clamp(max=self.post if self.post > 0 else max_len)[:, None]
        valid = pos < limit
        gidx = (keep.long() + offs[:-1, None].long())[valid]
        out_boxes, out_scores = boxes[gidx], scores[gidx]
        # modules/pyramid_proposal.py:61-67: final top-N over levels by score
        _, idx = torch.sort(-out_scores, dim=0, stable=True)
        idx = idx[:self.post]
        rois = torch.cat([torch.zeros((idx.numel(), 1), device=dev), out_boxes[idx]], 1)
        return rois, out_scores[idx]


class MaskROI:
    """operators/modules/mask_roi.py:24-146 on the device (decode, clip, per-class threshold + NMS,
    global top-`top_n`).  Output order = the reference's: class-major, NMS (descending score) order."""

    def __init__(self, top_n, num_classes, nms_thresh=0.5, class_agnostic=False, score_thresh=0.05,
                 bbox_reg_weights=(10., 10., 5., 5.)):
        self.top_n, self.num_classes = top_n, num_classes
        self.nms_thresh, self.class_agnostic, self.score_thresh = nms_thresh, class_agnostic, score_thresh
        self.weights = bbox_reg_weights

    def __call__(self, rois, bbox_delta, cls_prob, im_info):
        dev = rois.device
        C = self.num_classes
        proposal = bbox_transform(rois[:, 1:], bbox_delta, self.weights)
        proposal = clip_boxes(proposal, float(im_info[0]), float(im_info[1])).reshape(-1, C, 4)
        prob = cls_prob[:, 1:]                                    # skip background (j = 0)
        cand = prob > self.score_thresh
        ridx, cidx = torch.nonzero(cand, as_tuple=True)           # host sync (size); row-major = roi order
        if ridx.numel() == 0:                                     # mask_roi.py:132-139
            return (torch.ones(1, device=dev), torch.zeros(1, 5, device=dev),
                    torch.zeros(1, dtype=torch.long, device=dev))
        sc = prob[ridx, cidx]
        bx = proposal[ridx, cidx + 1]
        cls = cidx + 1
        seg_key = torch.zeros_like(cls) if self.class_agnostic else cls - 1
        nseg = 1 if self.class_agnostic else C - 1
        # order: segment ascending, score descending (stable => ties keep roi order)
        o1 = torch.sort(sc, descending=True, stable=True)[1]
        o2 = torch.sort(seg_key[o1], stable=True)[1]
        order = o1[o2]
        sc, bx, cls, seg_key = sc[order], bx[order], cls[order], seg_key[order]
        counts = torch.bincount(seg_key, minlength=nseg)
        offs = torch.zeros(nseg + 1, dtype=torch.int32, device=dev)
        offs[1:] = torch.cumsum(counts, 0).int()
        max_len = int(counts.max().item())                       # host sync (size)
        keep, cnt = nms_segmented(bx, offs, max_len, self.nms_thresh)
        pos = torch.arange(max_len, device=dev)[None, :]
        valid = pos < cnt[:, None]
        gidx = (keep.long() + offs[:-1, None].long())[valid]      # class-major, NMS order inside
        sc, bx, cls = sc[gidx], bx[gidx], cls[gidx]
        if self.top_n > 0 and sc.numel() > self.top_n:            # mask_roi.py:106-121
            thresh = torch.sort(sc)[0][-self.top_n]
            sel = sc >= thresh
            sc, bx, cls = sc[sel], bx[sel], cls[sel]
        boxes = torch.cat([torch.zeros((bx.shape[0], 1), device=dev), bx], 1)
        return sc, boxes, cls.long()


class PyramidProposal(torch.nn.Module):
    """operators/modules/pyramid_proposal.py:24-67 -- the reference's module signature on the device implementation:
    forward(cls_prob [5 x [B,A,h,w]], bbox_pred [5 x [B,4A,h,w]], im_info [B,3]) -> (rois [R,5], scores [R])."""

    def __init__(self, feat_stride, scales, ratios, rpn_pre_nms_top_n, rpn_post_nms_top_n, threshold, rpn_min_size,
                 individual_proposals=False, use_softnms=False):
        super().__init__()
        assert individual_proposals and not use_softnms, "the shipped configuration (config.py:123): per-level NMS, hard NMS"
        self.rpn_post_nms_top_n = rpn_post_nms_top_n
        self.gen = ProposalGenerator(tuple(int(s) for s in feat_stride), tuple(scales), tuple(ratios), rpn_pre_nms_top_n,
                                     rpn_post_nms_top_n, threshold, rpn_min_size)

    def forward(self, cls_prob, bbox_pred, im_info, roidb=None):
        assert roidb is None, "crowd filtering is a training-time option"
        im_info = np.asarray(im_info, dtype=np.float32).reshape(-1, 3)
        rois, scores = [], []
        for i in range(im_info.shape[0]):
            r, s = self.gen([c[[i]] for c in cls_prob], [b[[i]] for b in bbox_pred], im_info[i])
            r = r.clone(); r[:, 0] = i                                              # batch index column
            rois.append(r); scores.append(s)
        rois, scores = torch.cat(rois, 0), torch.cat(scores, 0)
        _, idx = torch.sort(-scores, dim=0, stable=True)                               # modules/pyramid_proposal.py:61-66
        idx = idx[:self.rpn_post_nms_top_n]
        return rois[idx, :], scores[idx]


class MaskROIModule(torch.nn.Module):
    """operators/modules/mask_roi.py:24-36 constructor + forward signature on the device implementation."""

    def __init__(self, clip_boxes, bbox_class_agnostic, top_n, num_classes, nms_thresh=None, class_agnostic=False,
                 score_thresh=None, bbox_reg_weights=(10., 10., 5., 5.)):
        super().__init__()
        assert clip_boxes and not bbox_class_agnostic, "the shipped configuration (resnet_upsnet.py:57-66)"
        self.impl = MaskROI(top_n, num_classes, 0.5 if nms_thresh is None else nms_thresh, class_agnostic,
                            0.05 if score_thresh is None else score_thresh, bbox_reg_weights)

    def forward(self, bottom_rois, bbox_delta, cls_prob, im_info, nms=True, cls_score=None, cls_label=None):
        assert nms and cls_score is None and cls_label is None, "inference call shape (resnet_upsnet.py:203,217)"
        info = np.asarray(im_info, dtype=np.float32).reshape(-1, 3)[0]
        return self.impl(bottom_rois, bbox_delta, cls_prob, info)


# ================================================================================================
# Static-shape, synchronisation-free variants (the engine path).  Same decisions as the classes above
# for every valid entry, but all outputs are padded to fixed sizes with a device-side count, so the
# whole forward can run without a host round trip and be captured in a CUDA graph
# (SURVEY.md section 8f rank 1; the reference synchronises >= 6 times per image, F8).
# ================================================================================================
NEG_INF = float("-inf")


class StaticProposalGenerator(ProposalGenerator):
    def _base_anchors(self, L, dev):
        key = ("base", L, str(dev))
        if key not in self._anchors:
            base = np.stack([generate_anchors(self.feat_stride[l], np.array(self.scales) * self.feat_stride[l], self.ratios)
                             for l in range(L)])
            self._anchors[key] = torch.from_numpy(np.ascontiguousarray(base, dtype=np.float64)).to(dev)
        return self._anchors[key]

    def _offsets(self, lens, dev):
        key = ("offs", tuple(lens), str(dev))
        if key not in self._anchors:
            self._anchors[key] = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=dev)
        return self._anchors[key]

    def __call__(self, cls_probs, bbox_preds, im_info):
        """im_info: the (h, w, scale) row, a float32 [3] tensor on the device of cls_probs or a host row (uploaded).
        -> rois [post,5] (invalid rows are all-zero), scores [post], valid [post] bool."""
        assert self.min_size == 0, "static path assumes config.test.rpn_min_size == 0 (all shipped yamls)"
        dev = cls_probs[0].device
        im_info = _ops.im_info_device(im_info, dev)
        im_h, im_w = im_info[0], im_info[1]
        boxes_l, scores_l, lens, idx_l = [], [], [], []
        fused = FUSED["on"] and dev.type == "cuda"
        if fused and 0 < self.pre <= 2048 and all(c.shape[0] == 1 and c.numel() < (1 << 22) for c in cls_probs):
            # one radix-select + sort for all levels, then one decode launch
            A = cls_probs[0].shape[1]
            scores, top_i, lens = _ops.rpn_topk([c[0] for c in cls_probs], A, self.pre)
            starts = np.concatenate([[0], np.cumsum(lens)])
            idx_l = [top_i[starts[l]:starts[l + 1]] for l in range(len(lens))]
            boxes = _ops.rpn_decode([b[0] for b in bbox_preds], idx_l, [c.shape[-2:] for c in cls_probs],
                                    self.feat_stride[:len(cls_probs)], self._base_anchors(len(cls_probs), dev), A, im_info)
            return self._after_topk(boxes, scores, lens, dev)
        for l in range(len(cls_probs)):
            A = cls_probs[l].shape[1]
            h, w = cls_probs[l].shape[-2:]
            scores = cls_probs[l][0].permute(1, 2, 0).reshape(-1)
            k = min(self.pre, scores.numel()) if self.pre > 0 else scores.numel()
            top_s, top_i = torch.topk(scores, k, sorted=True)
            scores_l.append(top_s); lens.append(k); idx_l.append(top_i)
            if not fused:
                deltas = bbox_preds[l][0].reshape(A, 4, h, w).permute(2, 3, 0, 1).reshape(-1, 4)
                boxes_l.append(clip_boxes(bbox_transform(self.anchors(l, h, w, dev)[top_i], deltas[top_i]), im_h, im_w))
        if fused:   # one launch: shifted anchors + bbox_transform + clip for the top-k of every level
            boxes = _ops.rpn_decode([b[0] for b in bbox_preds], idx_l, [c.shape[-2:] for c in cls_probs],
                                    self.feat_stride[:len(cls_probs)], self._base_anchors(len(cls_probs), dev),
                                    cls_probs[0].shape[1], im_info)
        else:
            boxes = torch.cat(boxes_l)
        scores = torch.cat(scores_l)
        return self._after_topk(boxes, scores, lens, dev)

    def _after_topk(self, boxes, scores, lens, dev):
        offs = self._offsets(lens, dev)
        max_len = max(lens)
        keep, cnt = nms_segmented(boxes, offs, max_len, self.thresh)
        if (FUSED["on"] and dev.type == "cuda" and 0 < self.post <= 2048 and len(lens) * min(max_len, self.post) <= 8192
                and len(lens) * min(max_len, self.post) >= self.post):
            return _ops.rpn_collect(keep, cnt, offs, boxes, scores, self.post)
        pos = torch.arange(max_len, device=dev)[None, :]
        limit = cnt.clamp(max=self.post if self.post > 0 else max_len)[:, None]
        valid = pos < limit
        gidx = (keep.long() + offs[:-1, None].long()).clamp_(0, boxes.shape[0] - 1)   # rows >= cnt are garbage
        sc = torch.where(valid, scores[gidx], torch.full_like(scores[gidx], NEG_INF))
        k = min(self.post, sc.numel())
        top_s, top_i = torch.topk(sc.reshape(-1), k, sorted=True)
        ok = top_s > NEG_INF
        sel = gidx.reshape(-1)[top_i]
        rois = torch.cat([torch.zeros((k, 1), device=dev), boxes[sel]], 1) * ok[:, None]
        return rois, torch.where(ok, top_s, torch.zeros_like(top_s)), ok


def _compact(values_list, flag, cap, dev):
    """Stable compaction of the rows where `flag` is set into `cap` slots (extra rows dropped).
    Returns ([compacted tensors], count int32 device scalar)."""
    n_all = flag.numel()
    dest = torch.cumsum(flag.to(torch.int64), 0) - 1
    count = flag.sum().clamp(max=cap).to(torch.int32)
    slot = torch.where(flag & (dest < cap), dest, torch.full_like(dest, cap))     # cap = dump slot
    outs = []
    for v in values_list:
        buf = torch.zeros((cap + 1,) + tuple(v.shape[1:]), dtype=v.dtype, device=dev)
        buf.index_copy_(0, slot, v[:n_all]) if False else buf.scatter_(
            0, slot.view(-1, *([1] * (v.dim() - 1))).expand_as(v), v)
        outs.append(buf[:cap])
    return outs, count


class StaticMaskROI(MaskROI):
    """MaskROI with fixed-size outputs: scores [cap], boxes [cap,5], cls [cap], n (int32 device scalar).
    cap = top_n + slack (ties at the top-n score threshold are all kept by the reference)."""

    def __init__(self, *a, slack=28, **kw):
        super().__init__(*a, **kw)
        self.cap = self.top_n + slack
        self.last_flags = None        # device int32 scalar of the last call: != 0 when the fixed-size buffers dropped detections
        self._const = {}

    def _consts(self, R, dev):
        key = (R, str(dev))
        if key not in self._const:
            Cm = self.num_classes - 1
            cls_flat = torch.arange(1, self.num_classes, device=dev).repeat(R)
            ridx_flat = torch.arange(R, device=dev).repeat_interleave(Cm)
            self._const[key] = (cls_flat, ridx_flat)
        return self._const[key]

    def __call__(self, rois, roi_valid, bbox_delta, cls_prob, im_info, side=False):
        """im_info: the (h, w, scale) row, a float32 [3] tensor on the rois' device or a host row (uploaded).
        side=True: this call runs on a side stream concurrently with another MaskROI (separate NMS scratch)."""
        dev = rois.device
        im_info = _ops.im_info_device(im_info, dev)
        C, R = self.num_classes, rois.shape[0]
        Cm = C - 1
        nseg = 1 if self.class_agnostic else Cm
        # a softmax row has at most one entry above 0.5, so class-agnostic candidates <= R when thresh >= 0.5
        M = R if (not self.class_agnostic or self.score_thresh >= 0.5) else R * Cm
        if FUSED["on"] and dev.type == "cuda" and R * Cm <= 8192 and Cm <= 128:
            sc, cls, bx, offs = _ops.maskroi_prepare(rois, roi_valid, bbox_delta, cls_prob, self.class_agnostic,
                                                     self.score_thresh, self.weights, im_info)
            keep, cnt = (_ops.nms_segmented(bx, offs, M, self.nms_thresh, side=True) if side
                         else nms_segmented(bx, offs, M, self.nms_thresh))
            o_sc, o_bx, o_cls, n_out, self.last_flags = _ops.maskroi_finish(keep, cnt, offs, sc, cls, bx, self.top_n, self.cap)
            return o_sc, o_bx, o_cls, n_out
        cls_flat, ridx_flat = self._consts(R, dev)
        proposal = clip_boxes(bbox_transform(rois[:, 1:], bbox_delta, self.weights), im_info[0],
                              im_info[1]).reshape(R, C, 4)
        prob = cls_prob[:, 1:]
        cand = ((prob > self.score_thresh) & roi_valid[:, None]).reshape(-1)
        sc_all = torch.where(cand, prob.reshape(-1), torch.full_like(prob.reshape(-1), -1.0))
        key = torch.where(cand, torch.zeros_like(cls_flat) if self.class_agnostic else cls_flat - 1,
                          torch.full_like(cls_flat, nseg))
        o1 = torch.sort(sc_all, descending=True, stable=True)[1]
        o2 = torch.sort(key[o1], stable=True)[1]
        order = o1[o2]
        sc, cls, key = sc_all[order], cls_flat[order], key[order]
        bx = proposal[ridx_flat[order], cls]
        counts = (key[:, None] == torch.arange(nseg, device=dev)[None, :]).sum(0)
        offs = torch.zeros(nseg + 1, dtype=torch.int32, device=dev)
        offs[1:] = torch.cumsum(counts, 0).to(torch.int32)
        keep, cnt = nms_segmented(bx, offs, M, self.nms_thresh)
        pos = torch.arange(M, device=dev)[None, :]
        valid = (pos < cnt[:, None]).reshape(-1)
        gidx = (keep.long() + offs[:-1, None].long()).clamp_(0, sc.numel() - 1).reshape(-1)
        # 1st compaction: class-major, NMS order inside (mask_roi.py:96-104)
        all_cap = min(nseg * M, 4096)
        (kidx,), nk = _compact([gidx], valid, all_cap, dev)
        n_surv = valid.sum()
        live = torch.arange(all_cap, device=dev) < nk
        ks = torch.where(live, sc[kidx], torch.full((all_cap,), NEG_INF, device=dev))
        # global top-n: keep scores >= the top_n-th largest (mask_roi.py:106-121); fewer than top_n => keep all
        kth = torch.topk(ks, min(self.top_n, all_cap), sorted=True)[0][-1] if self.top_n > 0 else NEG_INF
        sel = live & (ks >= kth)
        (oidx,), n_out = _compact([kidx], sel, self.cap, dev)
        # truncation flags like upsnet_maskroi_finish: bit 0 survivors beyond the candidate slots, bit 1 tie beyond the slack
        self.last_flags = ((n_surv > all_cap).to(torch.int32) + 2 * (sel.sum() > self.cap).to(torch.int32)).to(torch.int32)
        slot_live = torch.arange(self.cap, device=dev) < n_out
        out_sc = torch.where(slot_live, sc[oidx], torch.zeros(self.cap, device=dev))
        out_bx = torch.cat([torch.zeros((self.cap, 1), device=dev), bx[oidx]], 1) * slot_live[:, None]
        out_cls = torch.where(slot_live, cls[oidx], torch.zeros_like(cls[oidx]))
        # mask_roi.py:132-139: nothing survives -> one dummy detection (score 1, zero box, class 0)
        empty = n_out == 0
        out_sc[0] = torch.where(empty, 1.0, out_sc[0])
        n_out = torch.where(empty, torch.ones_like(n_out), n_out)
        return out_sc, out_bx, out_cls.long(), n_out
