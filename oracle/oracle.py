"""ctypes/numpy front-end of the CPU oracle (TEST INFRASTRUCTURE ONLY).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module; the product package ``upsnet_b200`` never does.

* C restatements (oracle/upsnet_oracle.c) are reached through ``libupsnet_oracle.so``.
* ``panoptic_head_literal`` is a second, line-by-line numpy restatement of the reference's
  python (mask_removal.py:29-93, unary_logits.py:78-105, resnet_upsnet.py:217-247) that
  materialises the [k,H,W] planes exactly like the reference does; it pins the fused C version
  at small sizes.
* ``RefKernels`` loads oracle/_ref/libupsnet_ref.so = the reference's own .cu kernels compiled
  for sm_90a (where the reference checkout is present).
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
i64p = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")


def build(force=False):
    """Compile the C oracle (and oracle/_ref when /root/reference exists)."""
    so = os.path.join(_HERE, "libupsnet_oracle.so")
    src = os.path.join(_HERE, "upsnet_oracle.c")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, os.path.join(_HERE, "libupsnet_oracle.so")])
    if os.path.isdir("/root/reference/upsnet/operators/src") and (
            force or not os.path.exists(os.path.join(_HERE, "_ref", "libupsnet_ref.so"))):
        from upsnet_b200.build import nvcc
        subprocess.check_call(["make", "-C", _HERE, "ref", "NVCC=" + nvcc()])
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        L = _LIB
        L.oracle_roi_align_forward.argtypes = [f32p, C.c_int, C.c_int, C.c_int, C.c_int, f32p, C.c_int,
                                               C.c_int, C.c_int, C.c_int, C.c_float, f32p]
        L.oracle_fpn_level.argtypes = [f32p, C.c_int, i32p]
        L.oracle_deform_conv_forward.argtypes = [f32p, f32p, C.c_void_p, f32p, C.c_void_p, f32p] + [C.c_int] * 14
        L.oracle_deform_conv_forward.restype = C.c_int
        L.oracle_deform_im2col.argtypes = [f32p, f32p, C.c_void_p] + [C.c_int] * 12 + [f32p]
        L.oracle_nms.argtypes = [f32p, C.c_int, C.c_float, i32p, i32p]
        L.oracle_bbox_transform.argtypes = [f32p, f32p, C.c_int, C.c_int] + [C.c_float] * 4 + [f32p]
        L.oracle_clip_boxes.argtypes = [f32p, C.c_int, C.c_float, C.c_float]
        L.oracle_mask_resize.argtypes = [f32p, C.c_int, C.c_int, f32p]
        L.oracle_panoptic_head.argtypes = [f32p, C.c_int, C.c_int, C.c_int, f32p, f32p, f32p, i64p, C.c_int,
                                           C.c_int, C.c_double, i64p, i32p, i64p, C.c_void_p]
        L.oracle_panoptic_head.restype = C.c_int
        L.oracle_conv2d.argtypes = [f32p, f32p, C.c_void_p, f32p] + [C.c_int] * 14
    return _LIB


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _optptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def conv_out(n, pad, dil, k, stride):
    return (n + 2 * pad - (dil * (k - 1) + 1)) // stride + 1


def roi_align(feat, rois, ph, pw, spatial_scale, sampling_ratio=2):
    feat, rois = _f32(feat), _f32(rois)
    B, Cc, H, W = feat.shape
    out = np.empty((rois.shape[0], Cc, ph, pw), np.float32)
    lib().oracle_roi_align_forward(feat, B, Cc, H, W, rois, rois.shape[0], ph, pw, sampling_ratio,
                                   spatial_scale, out)
    return out


def fpn_level(rois):
    rois = _f32(rois)
    lv = np.empty(rois.shape[0], np.int32)
    lib().oracle_fpn_level(rois, rois.shape[0], lv)
    return lv


def fpn_level_numpy(rois):
    """fpn_roi_align.py:35-38 verbatim (float32 numpy)."""
    rois = _f32(rois)
    w = rois[:, 3] - rois[:, 1] + 1
    h = rois[:, 4] - rois[:, 2] + 1
    return np.clip(np.floor(2 + np.log2(np.sqrt(w * h) / 224 + 1e-6)), 0, 3).astype(np.int32)


def fpn_roi_align(feats, rois, ph, pw, scales=(1 / 4., 1 / 8., 1 / 16., 1 / 32.)):
    """FPNRoIAlign.forward (fpn_roi_align.py:32-62): per-level ROIAlign, results in roi order."""
    rois = _f32(rois)
    lv = fpn_level_numpy(rois)
    out = np.zeros((rois.shape[0], feats[0].shape[1], ph, pw), np.float32)
    for l in range(4):
        idx = np.where(lv == l)[0]
        if len(idx):
            out[idx] = roi_align(feats[l], rois[idx], ph, pw, scales[l])
    return out


def deform_conv(x, offset, weight, bias=None, mask=None, stride=1, pad=0, dil=1, dg=1):
    """DeformConvFunction.forward (functions/deform_conv.py:26-57); mask!=None -> v2
    (functions/mod_deform_conv.py:25-59; mask is the already-activated 2*sigmoid(m))."""
    x, offset, weight = _f32(x), _f32(offset), _f32(weight)
    N, Cin, H, W = x.shape
    Cout, _, kh, kw = weight.shape
    Ho, Wo = conv_out(H, pad, dil, kh, stride), conv_out(W, pad, dil, kw, stride)
    y = np.empty((N, Cout, Ho, Wo), np.float32)
    b = None if bias is None else _f32(bias)
    m = None if mask is None else _f32(mask)
    rc = lib().oracle_deform_conv_forward(x, offset, _optptr(m), weight.reshape(Cout, -1), _optptr(b), y,
                                          N, Cin, H, W, Cout, kh, kw, stride, stride, pad, pad, dil, dil, dg)
    assert rc == 0
    return y


def mod_deform_conv(x, offset_mask, weight, bias=None, stride=1, pad=0, dil=1, dg=1):
    """ModDeformConv.forward (modules/mod_deform_conv.py:60-67): chunk -> offset, mask=2*sigmoid."""
    om = _f32(offset_mask)
    o1, o2, m = np.split(om, 3, axis=1)
    offset = np.concatenate([o1, o2], axis=1)
    mask = (1.0 / (1.0 + np.exp(-m.astype(np.float64))) * 2).astype(np.float32)
    return deform_conv(x, offset, weight, bias, mask, stride, pad, dil, dg)


def conv2d(x, weight, bias=None, stride=1, pad=0, dil=1, relu=False):
    x, weight = _f32(x), _f32(weight)
    N, Cin, H, W = x.shape
    Cout, _, kh, kw = weight.shape
    Ho, Wo = conv_out(H, pad, dil, kh, stride), conv_out(W, pad, dil, kw, stride)
    y = np.empty((N, Cout, Ho, Wo), np.float32)
    b = None if bias is None else _f32(bias)
    lib().oracle_conv2d(x, weight, _optptr(b), y, N, Cin, H, W, Cout, kh, kw, stride, stride, pad, pad,
                        dil, dil, int(relu))
    return y


def nms(dets, thresh):
    """gpu_nms(dets, thresh) -> list[int] of original indices, descending score."""
    dets = _f32(dets)
    n = dets.shape[0]
    keep = np.empty(max(n, 1), np.int32)
    num = np.zeros(1, np.int32)
    lib().oracle_nms(dets.reshape(-1, 5) if n else np.zeros((1, 5), np.float32), n, thresh, keep, num)
    return keep[:num[0]].tolist()


def bbox_transform(boxes, deltas, weights=(1., 1., 1., 1.)):
    boxes, deltas = _f32(boxes), _f32(deltas)
    out = np.empty_like(deltas)
    lib().oracle_bbox_transform(boxes, deltas, boxes.shape[0], deltas.shape[1] // 4, *weights, out)
    return out


def clip_boxes(boxes, im_shape):
    boxes = _f32(boxes).copy()
    lib().oracle_clip_boxes(boxes, boxes.size // 4, float(im_shape[0]), float(im_shape[1]))
    return boxes


def mask_resize(S, w, h):
    S = _f32(S).reshape(28, 28)
    out = np.empty((h, w), np.float32)
    lib().oracle_mask_resize(S, w, h, out)
    return out


def panoptic_head(fcn, boxes, cls_prob, mask_logit, cls_idx, num_stuff, fraction_threshold=0.3,
                  want_sem=False):
    """Fused C restatement.  fcn [S,H,W]; boxes [n,4]; mask_logit [n,28,28]; cls_idx [n] int64."""
    fcn = _f32(fcn)
    S, H, W = fcn.shape
    n = int(boxes.shape[0])
    boxes, cls_prob, mask_logit = _f32(boxes).reshape(-1, 4), _f32(cls_prob).reshape(-1), _f32(mask_logit).reshape(-1, 28, 28)
    cls_idx = np.ascontiguousarray(cls_idx, np.int64).reshape(-1)
    keep = np.zeros(max(n, 1), np.int64)
    k = np.zeros(1, np.int32)
    labels = np.empty((H, W), np.int64)
    sem = np.empty((H, W), np.int64) if want_sem else None
    rc = lib().oracle_panoptic_head(fcn, S, H, W, boxes, cls_prob, mask_logit, cls_idx, n, num_stuff,
                                    fraction_threshold, keep, k, labels, _optptr(sem))
    assert rc == 0
    return (keep[:k[0]].copy(), labels) + ((sem,) if want_sem else ())


# ---------------------------------------------------------------------------------------------
# Line-by-line numpy restatement (materialises planes like the reference).  resize = either the
# oracle-of-record formula (default) or real cv2.resize (informational, needs cv2).
# ---------------------------------------------------------------------------------------------
def panoptic_head_literal(fcn, boxes, cls_prob, mask_logit, cls_idx, num_stuff, fraction_threshold=0.3,
                          resize="formula", return_logits=False):
    fcn = _f32(fcn)
    S, H, W = fcn.shape
    im_shape = (H, W)
    mask_rois = _f32(boxes).reshape(-1, 4)
    cls_prob = _f32(cls_prob).reshape(-1)
    mask_logit_all = _f32(mask_logit).reshape(-1, 28, 28)
    cls_idx0 = np.asarray(cls_idx, np.int64).reshape(-1)

    def do_resize(src, w, h):
        if resize == "cv2":
            import cv2
            return cv2.resize(src, (w, h))
        return mask_resize(src, w, h)

    # ---- MaskRemoval.forward (mask_removal.py:43-93) ----
    n = mask_rois.shape[0]
    mask_energy = np.zeros((1, n, H, W), np.float32)
    frame_id = 0
    mask_image = np.zeros((int(np.max(cls_idx0)),) + im_shape, dtype=np.uint8)
    # stable-desc tie rule (reference: np.argsort(cls_prob)[::-1], unspecified on ties)
    sorted_inds = np.lexsort((np.arange(n), -cls_prob.astype(np.float64)))
    mr = mask_rois[sorted_inds]
    ml = mask_logit_all[sorted_inds]
    ci = cls_idx0[sorted_inds] - 1
    keep_inds = []
    dummy = (len(ci) == 1 and ci[0] == -1)
    if not dummy:
        ref_boxes = mr.astype(np.int32)
        for i in range(n):
            ref_box = ref_boxes[i, :]
            w = max(ref_box[2] - ref_box[0] + 1, 1)
            h = max(ref_box[3] - ref_box[1] + 1, 1)
            logit = do_resize(ml[i], int(w), int(h))
            mask = np.array(logit > 0, dtype=np.uint8)
            x_0 = max(ref_box[0], 0)
            x_1 = min(ref_box[2] + 1, im_shape[1])
            y_0 = max(ref_box[1], 0)
            y_1 = min(ref_box[3] + 1, im_shape[0])
            crop_mask = mask[(y_0 - ref_box[1]):(y_1 - ref_box[1]), (x_0 - ref_box[0]):(x_1 - ref_box[0])]
            mask_sum = crop_mask.sum()
            mask_image_crop = mask_image[ci[i]][y_0:y_1, x_0:x_1]
            if mask_sum == 0 or (np.logical_and(mask_image_crop >= 1, crop_mask == 1).sum() / mask_sum
                                 > fraction_threshold):
                continue
            keep_inds.append(int(sorted_inds[i]))
            mask_image[ci[i]][y_0:y_1, x_0:x_1] += crop_mask
            mask_energy[0, frame_id, y_0:y_1, x_0:x_1] = \
                logit[(y_0 - ref_box[1]):(y_1 - ref_box[1]), (x_0 - ref_box[0]):(x_1 - ref_box[0])]
            frame_id += 1
    mask_energy = mask_energy[:, :len(keep_inds)]
    if len(keep_inds) == 0:
        mask_energy = np.zeros((1, 1, H, W), np.float32)
        keep_inds = [0]
    keep = np.array(keep_inds, np.int64)

    # ---- glue (resnet_upsnet.py:224-227) + SegTerm.forward (unary_logits.py:85-105) ----
    k_rois = np.concatenate([np.zeros((len(keep), 1), np.float32), mask_rois[keep]], 1) * np.float32(4.0)
    k_cls = cls_idx0[keep]
    seg_logits = fcn[None, :num_stuff]
    b = k_rois[:, 1:] * np.float32(0.25)
    seg_inst = np.zeros((1, len(keep), H, W), np.float32)
    for i in range(len(keep)):
        if k_cls[i] == 0:
            continue
        y0 = int(b[i][1]); y1 = int(b[i][3].round() + 1)
        x0 = int(b[i][0]); x1 = int(b[i][2].round() + 1)
        seg_inst[0, i, y0:y1, x0:x1] = fcn[num_stuff + k_cls[i] - 1, y0:y1, x0:x1]

    # ---- resnet_upsnet.py:234-240 ----
    void_logits = fcn[None, num_stuff:].max(axis=1, keepdims=True) - seg_inst.max(axis=1, keepdims=True)
    inst_logits = seg_inst + mask_energy
    panoptic_logits = np.concatenate([seg_logits, inst_logits, void_logits], axis=1)
    void_id = panoptic_logits.shape[1] - 1
    out = panoptic_logits.argmax(axis=1)[0].astype(np.int64)
    out[out == void_id] = 255
    if return_logits:
        return keep, out, panoptic_logits[0]
    return keep, out


def unified_pan_result(seg, pan, cls_ind, num_seg_classes, num_classes, stuff_area_limit=4 * 64 * 64):
    """dataset/base_dataset.py:332-371 get_unified_pan_result for ONE image, restated with explicit histograms (the
    reference uses np.unique per segment).  seg / pan [H,W] ints, cls_ind [k] -> uint8 [H,W,3]."""
    seg, pan = np.asarray(seg), np.asarray(pan)
    id_last = num_seg_classes - num_classes
    pan_seg = pan.copy()
    pan_ins = np.where(pan <= id_last, 0, pan)
    ids = np.unique(pan)
    ids_ins = ids[ids > id_last]
    for idx, i in enumerate(ids_ins):
        region = pan == i
        if i == 255:
            pan_seg[region] = 255
            pan_ins[region] = 0
            continue
        cnt = np.bincount(seg[region].astype(np.int64), minlength=num_seg_classes)
        major = int(np.argmax(cnt))                                     # first maximum = smallest class id
        target = int(cls_ind[i - id_last - 1]) + id_last
        if major != target and 2 * int(cnt.max()) >= int(cnt.sum()) and major <= id_last:
            pan_seg[region] = major
            pan_ins[region] = 0
        else:
            pan_seg[region] = target
            pan_ins[region] = idx + 1
    for c in np.unique(pan_seg):
        if c <= id_last and (pan_seg == c).sum() < stuff_area_limit:
            pan_seg[pan_seg == c] = 255
    out = np.zeros(pan.shape + (3,), np.uint8)
    out[..., 0] = pan_seg
    out[..., 1] = pan_ins
    return out


def prep_image(im_hwc_u8, pixel_means, scale, stride=32):
    """dataset/base_dataset.py:143-174 + :898-923 for one target size: float32, mean subtraction, cv2.resize by `scale`
    (INTER_LINEAR), CHW, zero padding to a multiple of `stride`.  Uses the real cv2 (what the reference calls)."""
    import cv2
    im = im_hwc_u8.astype(np.float32, copy=True)
    im -= np.asarray(pixel_means, np.float64).reshape((1, 1, -1))      # float64 means: numpy subtracts in double, stores float32
    im = cv2.resize(im, None, None, fx=scale, fy=scale, interpolation=cv2.INTER_LINEAR)
    chw = im.transpose(2, 0, 1)
    Hp = int(np.ceil(chw.shape[1] / float(stride)) * stride)
    Wp = int(np.ceil(chw.shape[2] / float(stride)) * stride)
    blob = np.zeros((1, 3, Hp, Wp), np.float32)
    blob[0, :, :chw.shape[1], :chw.shape[2]] = chw
    return blob, chw.shape[1:]


class RefKernels:
    """The reference's own CUDA kernels (oracle/_ref/libupsnet_ref.so), torch tensors in/out."""

    def __init__(self):
        path = os.path.join(_HERE, "_ref", "libupsnet_ref.so")
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        self.L = C.CDLL(path)
        vp = C.c_void_p
        self.L.ref_roi_align_forward.argtypes = [vp, C.c_float] + [C.c_int] * 7 + [vp, vp, vp]
        self.L.ref_deform_im2col.argtypes = [vp, vp] + [C.c_int] * 12 + [vp, vp]
        self.L.ref_mod_deform_im2col.argtypes = [vp, vp, vp] + [C.c_int] * 14 + [vp, vp]
        self.L.ref_nms.argtypes = [i32p, i32p, f32p, C.c_int, C.c_float, C.c_int]

    @staticmethod
    def _stream():
        import torch
        return torch.cuda.current_stream().cuda_stream

    def roi_align(self, feat, rois, ph, pw, scale, sr=2):
        import torch
        feat, rois = feat.contiguous().float(), rois.contiguous().float()
        out = torch.zeros(rois.shape[0], feat.shape[1], ph, pw, device=feat.device)
        rc = self.L.ref_roi_align_forward(feat.data_ptr(), scale, rois.shape[0], feat.shape[2], feat.shape[3],
                                          feat.shape[1], ph, pw, sr, rois.data_ptr(), out.data_ptr(),
                                          self._stream())
        assert rc == 0
        return out

    def deform_conv(self, x, offset, weight, bias=None, mask=None, stride=1, pad=0, dil=1, dg=1):
        """functions/deform_conv.py:44-57 with the reference im2col kernel + torch.mm."""
        import torch
        x, offset = x.contiguous().float(), offset.contiguous().float()
        N, Cin, H, W = x.shape
        Cout, _, kh, kw = weight.shape
        Ho, Wo = conv_out(H, pad, dil, kh, stride), conv_out(W, pad, dil, kw, stride)
        col = torch.zeros(Cin * kh * kw, Ho * Wo, device=x.device)
        y = torch.zeros(N, Cout, Ho, Wo, device=x.device)
        for i in range(N):
            if mask is None:
                rc = self.L.ref_deform_im2col(x[i].data_ptr(), offset[i].data_ptr(), Cin, H, W, kh, kw, pad, pad,
                                              stride, stride, dil, dil, dg, col.data_ptr(), self._stream())
            else:
                m = mask.contiguous().float()
                rc = self.L.ref_mod_deform_im2col(x[i].data_ptr(), offset[i].data_ptr(), m[i].data_ptr(), Cin, H,
                                                  W, Ho, Wo, kh, kw, pad, pad, stride, stride, dil, dil, dg,
                                                  col.data_ptr(), self._stream())
            assert rc == 0
            y[i] = torch.mm(weight.reshape(Cout, -1).float(), col).view(Cout, Ho, Wo)
        if bias is not None:
            y += bias.view(1, -1, 1, 1)
        return y

    def nms(self, dets, thresh, device_id=0):
        """gpu_nms.pyx:23-38: host argsort desc, _nms on sorted boxes, order[keep]."""
        dets = _f32(dets)
        n = dets.shape[0]
        order = np.lexsort((np.arange(n), -dets[:, 4].astype(np.float64)))
        sorted_dets = np.ascontiguousarray(dets[order])
        keep = np.zeros(n, np.int32)
        num = np.zeros(1, np.int32)
        self.L.ref_nms(keep, num, sorted_dets, n, thresh, device_id)
        return order[keep[:num[0]]].tolist()


# ---------------------------------------------------------------------------------------------
# Row f4: im_post (upsnet_end2end_test.py:95-152) -- mask paste + COCO RLE.  Plain numpy restatement.
# The RLE codec is pycocotools' (cocoapi common/maskApi.c rleEncode / rleToString / rleFrString; the reference imports
# `pycocotools.mask.encode` at upsnet_end2end_test.py:48 without pinning a version; the package is not in this image):
# restated from its published algorithm -- "parity unpinned" for the codec itself, the paste semantics are pinned to the
# reference's own im_post executed with real cv2 (tests/golden/make_reference_impost.py).
# ---------------------------------------------------------------------------------------------
def resize_linear(src, w, h):
    """cv2.resize(src, (w, h)) for a float32 image, INTER_LINEAR, OpenCV's documented formula in un-fused float32
    (SURVEY A.5): float64 scale, float32 source coordinate; columns clamp the tap and zero the fraction at both borders,
    rows clamp the taps only; horizontal pass first."""
    src = _f32(src)
    sh, sw = src.shape

    def coef(n_dst, n_src):
        scale = np.float64(n_src) / np.float64(n_dst)
        f = ((np.arange(n_dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
        s = np.floor(f).astype(np.int32)
        return s, (f - s.astype(np.float32)).astype(np.float32)
    sx, fx = coef(w, sw)
    lo, hi = sx < 0, sx >= sw - 1
    sx[lo] = 0; fx[lo] = 0
    sx[hi] = sw - 1; fx[hi] = 0
    sx1 = np.minimum(sx + 1, sw - 1)
    sy, fy = coef(h, sh)
    y0, y1 = np.clip(sy, 0, sh - 1), np.clip(sy + 1, 0, sh - 1)
    a0 = (np.float32(1) - fx).astype(np.float32)
    hrow = (src[:, sx] * a0 + src[:, sx1] * fx).astype(np.float32)            # [sh, w]
    b0 = (np.float32(1) - fy).astype(np.float32)[:, None]
    return (hrow[y0] * b0 + hrow[y1] * fy[:, None]).astype(np.float32)


def expand_boxes(boxes, scale):
    """bbox/bbox_transform.py:365-381 on float32 boxes (the arithmetic stays float32, the result array is float64)."""
    boxes = _f32(boxes).reshape(-1, 4)
    w_half = (boxes[:, 2] - boxes[:, 0]) * np.float32(.5)
    h_half = (boxes[:, 3] - boxes[:, 1]) * np.float32(.5)
    x_c = (boxes[:, 2] + boxes[:, 0]) * np.float32(.5)
    y_c = (boxes[:, 3] + boxes[:, 1]) * np.float32(.5)
    w_half = w_half * np.float32(scale)
    h_half = h_half * np.float32(scale)
    out = np.zeros(boxes.shape)
    out[:, 0] = x_c - w_half; out[:, 2] = x_c + w_half
    out[:, 1] = y_c - h_half; out[:, 3] = y_c + h_half
    return out


def im_post_masks(pred_boxes, pred_masks, cls_inds, im_h, im_w, resize="formula"):
    """The [n, im_h, im_w] uint8 images im_post pastes (upsnet_end2end_test.py:100-139), detection order (not per class).
    pred_boxes [n,4]; pred_masks [n,C,M,M] probabilities; cls_inds [n]."""
    pred_masks = _f32(pred_masks)
    n, C, M, _ = pred_masks.shape
    ref = expand_boxes(pred_boxes, (M + 2.0) / M).astype(np.int32)
    out = np.zeros((n, im_h, im_w), np.uint8)
    padded = np.zeros((M + 2, M + 2), np.float32)
    for i in range(n):
        padded[1:-1, 1:-1] = pred_masks[i, int(cls_inds[i]) if C > 1 else 0]
        rb = ref[i]
        w = max(int(rb[2] - rb[0] + 1), 1); h = max(int(rb[3] - rb[1] + 1), 1)
        if resize == "cv2":
            import cv2
            m = cv2.resize(padded, (w, h))
        else:
            m = resize_linear(padded, w, h)
        m = np.array(m > 0.5, dtype=np.uint8)
        x_0, x_1 = max(int(rb[0]), 0), min(int(rb[2]) + 1, im_w)
        y_0, y_1 = max(int(rb[1]), 0), min(int(rb[3]) + 1, im_h)
        if x_1 > x_0 and y_1 > y_0:
            out[i, y_0:y_1, x_0:x_1] = m[(y_0 - rb[1]):(y_1 - rb[1]), (x_0 - rb[0]):(x_1 - rb[0])]
    return out


def rle_counts(mask):
    """maskApi.c rleEncode: run lengths of the column-major (Fortran) flattening, starting with the zeros run."""
    v = np.asarray(mask, np.uint8).flatten(order="F")
    if v.size == 0:
        return np.zeros(0, np.uint32)
    change = np.flatnonzero(v[1:] != v[:-1]) + 1
    edges = np.concatenate([[0], change, [v.size]])
    cnts = np.diff(edges)
    if v[0] != 0:
        cnts = np.concatenate([[0], cnts])
    return cnts.astype(np.uint32)


def rle_to_string(cnts):
    """maskApi.c rleToString: LEB128-like, 5 data bits per character, differences against the count two back."""
    out = bytearray()
    cnts = [int(c) for c in cnts]
    for i, x in enumerate(cnts):
        if i > 2:
            x -= cnts[i - 2]
        more = True
        while more:
            c = x & 0x1f
            x >>= 5
            more = (x != -1) if (c & 0x10) else (x != 0)
            if more:
                c |= 0x20
            out.append(c + 48)
    return bytes(out)


def rle_from_string(s):
    """maskApi.c rleFrString (inverse of rle_to_string)."""
    if isinstance(s, str):
        s = s.encode()
    cnts, p = [], 0
    while p < len(s):
        x, k, more = 0, 0, True
        while more:
            c = s[p] - 48
            x |= (c & 0x1f) << (5 * k)
            more = bool(c & 0x20)
            p += 1; k += 1
            if not more and (c & 0x10):
                x |= -1 << (5 * k)
        if len(cnts) > 2:
            x += cnts[-2]
        cnts.append(x)
    return np.asarray(cnts, np.uint32)


def rle_decode(cnts, h, w):
    v = np.zeros(h * w, np.uint8)
    p, val = 0, 0
    for c in cnts:
        c = int(c)
        if val:
            v[p:p + c] = 1
        p += c; val ^= 1
    return v.reshape((h, w), order="F")


def mask_encode(mask):
    """pycocotools.mask.encode for one [H,W] (or [H,W,1]) uint8 mask: {'size': [H,W], 'counts': bytes}."""
    m = np.asarray(mask)
    if m.ndim == 3:
        m = m[:, :, 0]
    return {"size": [int(m.shape[0]), int(m.shape[1])], "counts": rle_to_string(rle_counts(m))}
