"""CPU suite (-m "not gpu"): pins the oracle against the committed golden vectors (generated from
the reference's own python by tests/golden/make_golden.py), against torchvision, and checks host
logic + that the C-ABI library exports every symbol include/upsnet_b200.h declares."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_oracle_nms_matches_reference_py_cpu_nms(golden_ref):
    g = golden_ref
    for i in range(int(g["nms_cases"])):
        keep = O.nms(g["nms%d_dets" % i], float(g["nms%d_thresh" % i]))
        assert keep == g["nms%d_keep" % i].tolist(), "case %d" % i


def test_oracle_nms_edge_cases():
    assert O.nms(np.zeros((0, 5), np.float32), 0.5) == []
    d = np.array([[0, 0, 10, 10, 0.9], [0, 0, 10, 10, 0.8], [20, 20, 30, 30, 0.7]], np.float32)
    assert O.nms(d, 0.5) == [0, 2]
    # IoU == thresh is NOT suppressed (GPU / py semantics `>`, SURVEY F10): two 10x20 boxes sharing half
    d = np.array([[0, 0, 9, 19, 0.9], [0, 10, 9, 29, 0.8]], np.float32)  # inter 100, union 300 -> 1/3
    assert O.nms(d, 1.0 / 3.0 + 1e-3) == [0, 1]
    assert O.nms(d, 0.3) == [0]


def test_oracle_bbox_transform_matches_reference(golden_ref):
    g = golden_ref
    pred = O.bbox_transform(g["bt_boxes"], g["bt_deltas"], (10., 10., 5., 5.))
    np.testing.assert_allclose(pred, g["bt_pred"], rtol=1e-5, atol=1e-3)
    np.testing.assert_allclose(O.clip_boxes(g["bt_pred"], (600, 900)), g["bt_clipped"], rtol=0, atol=0)
    np.testing.assert_allclose(O.bbox_transform(g["bt_boxes"], g["bt_deltas"][:, :4]), g["bt_pred_w1"],
                               rtol=1e-5, atol=1e-3)


def test_oracle_roi_align_golden_and_torchvision(golden_ops):
    g = golden_ops
    out = O.roi_align(g["ra_feat"], g["ra_rois"], 7, 7, 0.25)
    assert np.array_equal(out, g["ra_out"])
    assert float(g["ra_tv_maxdiff"]) < 1e-5
    import torchvision
    tv = torchvision.ops.roi_align(torch.from_numpy(g["ra_feat"]), torch.from_numpy(g["ra_rois"]), (7, 7), 0.25, 2,
                                   False).numpy()
    assert np.abs(out - tv).max() < 1e-5
    # 14x14 variant + adaptive sampling ratio
    out14 = O.roi_align(g["ra_feat"], g["ra_rois"], 14, 14, 0.25)
    tv14 = torchvision.ops.roi_align(torch.from_numpy(g["ra_feat"]), torch.from_numpy(g["ra_rois"]), (14, 14), 0.25,
                                     2, False).numpy()
    assert np.abs(out14 - tv14).max() < 1e-5


def test_oracle_dcn_golden_and_torchvision(golden_ops):
    g = golden_ops
    y = O.deform_conv(g["dcn_x"], g["dcn_off"], g["dcn_w"], g["dcn_b"], pad=1, dg=2)
    np.testing.assert_allclose(y, g["dcn_y"], rtol=0, atol=1e-6)
    y2 = O.mod_deform_conv(g["dcn_x"], g["dcn2_om"], g["dcn_w"], g["dcn_b"], pad=1, dg=1)
    np.testing.assert_allclose(y2, g["dcn2_y"], rtol=0, atol=1e-6)
    assert float(g["dcn_tv_maxdiff"]) < 1e-5 and float(g["dcn2_tv_maxdiff"]) < 1e-5
    import torchvision
    x = torch.from_numpy(g["dcn_x"])
    for stride, pad, dil in [(1, 1, 1), (2, 1, 1), (1, 2, 2)]:
        Ho = O.conv_out(14, pad, dil, 3, stride); Wo = O.conv_out(18, pad, dil, 3, stride)
        off = (np.random.default_rng(stride * 10 + dil).standard_normal((2, 18, Ho, Wo)) * 1.5).astype(np.float32)
        yy = O.deform_conv(g["dcn_x"], off, g["dcn_w"], None, stride=stride, pad=pad, dil=dil)
        tv = torchvision.ops.deform_conv2d(x, torch.from_numpy(off), torch.from_numpy(g["dcn_w"]), None,
                                           stride=stride, padding=pad, dilation=dil).numpy()
        assert np.abs(yy - tv).max() < 1e-5


def test_oracle_conv2d_vs_torch():
    rng = np.random.default_rng(3)
    x = rng.standard_normal((2, 5, 11, 13)).astype(np.float32)
    w = rng.standard_normal((7, 5, 3, 3)).astype(np.float32) * 0.2
    b = rng.standard_normal(7).astype(np.float32)
    for stride, pad, dil in [(1, 1, 1), (2, 1, 1), (1, 2, 2), (2, 0, 1)]:
        y = O.conv2d(x, w, b, stride, pad, dil, relu=True)
        t = torch.relu(torch.nn.functional.conv2d(torch.from_numpy(x), torch.from_numpy(w), torch.from_numpy(b),
                                                  stride, pad, dil)).numpy()
        assert np.abs(y - t).max() < 1e-5


def test_oracle_panoptic_golden_and_literal(golden_ops):
    g = golden_ops
    keep, labels = O.panoptic_head(g["pan_fcn"], g["pan_boxes"], g["pan_prob"], g["pan_ml"], g["pan_cls"], 11)
    assert np.array_equal(keep, g["pan_keep"]) and np.array_equal(labels, g["pan_labels"])
    k2, l2 = O.panoptic_head_literal(g["pan_fcn"], g["pan_boxes"], g["pan_prob"], g["pan_ml"], g["pan_cls"], 11)
    assert np.array_equal(keep, k2) and np.array_equal(labels, l2)
    # informational: agreement with the real cv2.resize path recorded at generation time
    assert bool(g["pan_cv2_keep_equal"]) and int(g["pan_cv2_label_diff"]) <= 8


def _pan_case(n, H, W, seed, S=19, nthing=8):
    rng = np.random.default_rng(seed)
    fcn = (rng.standard_normal((S, H, W)) * 3).astype(np.float32)
    c = np.stack([rng.uniform(0, W, n), rng.uniform(0, H, n)], 1)
    s = np.exp(rng.uniform(np.log(6), np.log(min(H, W) / 2), (n, 2)))
    b = np.concatenate([c - s / 2, c + s / 2], 1).astype(np.float32)
    b[:, 0::2] = np.clip(b[:, 0::2], 0, W - 1); b[:, 1::2] = np.clip(b[:, 1::2], 0, H - 1)
    prob = (0.6 + 0.4 * (rng.permutation(n) + 1) / (n + 1)).astype(np.float32)
    ml = (rng.standard_normal((n, 28, 28)) * 2 + 0.5).astype(np.float32)
    cls = rng.integers(1, nthing + 1, n).astype(np.int64)
    return fcn, b, prob, ml, cls


@pytest.mark.parametrize("n,H,W", [(1, 40, 56), (7, 64, 96), (33, 80, 120)])
def test_oracle_panoptic_fused_equals_literal(n, H, W):
    fcn, b, prob, ml, cls = _pan_case(n, H, W, seed=n)
    k1, l1 = O.panoptic_head(fcn, b, prob, ml, cls, 11)
    k2, l2 = O.panoptic_head_literal(fcn, b, prob, ml, cls, 11)
    assert np.array_equal(k1, k2) and np.array_equal(l1, l2)


def test_oracle_panoptic_edge_cases():
    fcn, b, prob, ml, cls = _pan_case(3, 40, 56, seed=5)
    # all mask logits negative -> nothing kept -> reference fallback keep=[0], zero mask plane
    k1, l1 = O.panoptic_head(fcn, b, prob, -np.abs(ml) - 1, cls, 11)
    k2, l2 = O.panoptic_head_literal(fcn, b, prob, -np.abs(ml) - 1, cls, 11)
    assert k1.tolist() == [0] and np.array_equal(k1, k2) and np.array_equal(l1, l2)
    # identical boxes of one class: the second is pruned by the 0.3 overlap rule
    b2 = np.stack([b[0], b[0], b[1]]); cls2 = np.array([3, 3, 5]); ml2 = np.stack([ml[0], ml[0], ml[1]])
    k1, l1 = O.panoptic_head(fcn, b2, prob, ml2, cls2, 11)
    k2, l2 = O.panoptic_head_literal(fcn, b2, prob, ml2, cls2, 11)
    assert len(k1) == 2 and np.array_equal(k1, k2) and np.array_equal(l1, l2)


def test_mask_resize_close_to_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(9)
    S = (rng.standard_normal((28, 28)) * 2).astype(np.float32)
    for (w, h) in [(28, 28), (57, 91), (13, 9), (200, 130)]:
        a = O.mask_resize(S, w, h)
        ref = cv2.resize(S, (w, h))
        assert np.abs(a - ref).max() < 2e-5  # SURVEY A.5: cv2's float path is not bit-reproducible


def test_fpn_level_thresholds_match_numpy():
    """The CUDA kernel maps x = sqrt(w*h)/224+1e-6 to a level with the constants 0.5, 1.0, 0x3fffffff
    (roi_align.cu fpn_level_of).  Pin them against numpy's float32 evaluation of fpn_roi_align.py:37."""
    def lvl(x):
        return np.clip(np.floor(np.float32(2) + np.log2(np.asarray(x, np.float32))), 0, 3)
    thr = np.array([0x3f000000, 0x3f800000, 0x3fffffff], np.uint32)
    for k, t in enumerate(thr, start=1):
        bits = np.arange(int(t) - 256, int(t) + 256, dtype=np.uint32)
        l = lvl(bits.view(np.float32))
        assert (l[:256] < k).all() and (l[256:] >= k).all()
    rng = np.random.default_rng(1)
    rois = np.concatenate([np.zeros((5000, 1)), rng.uniform(0, 500, (5000, 2)), rng.uniform(500, 2000, (5000, 2))], 1)
    rois = rois.astype(np.float32)
    w = rois[:, 3] - rois[:, 1] + 1; h = rois[:, 4] - rois[:, 2] + 1
    x = (np.sqrt(w * h) / 224 + 1e-6).astype(np.float32)
    thr_f = thr.view(np.float32)
    mine = (x >= thr_f[0]).astype(int) + (x >= thr_f[1]) + (x >= thr_f[2])
    assert np.array_equal(mine, O.fpn_level_numpy(rois))
    assert np.array_equal(O.fpn_level(rois), O.fpn_level_numpy(rois))


def test_cabi_bindings_cover_every_declared_symbol(tmp_path):
    from upsnet_b200 import _lib, build
    header = open(os.path.join(ROOT, "include", "upsnet_b200.h")).read()
    declared = sorted(set(re.findall(r"\bint\s+(upsnet_\w+)\s*\(", header)))
    assert declared, "no declarations parsed"
    decls = dict(_lib.declarations())
    assert sorted(decls) == declared
    so = build.build()  # nvcc cross-compiles for sm_90a without a GPU
    L = ctypes.CDLL(so)
    for name in declared:
        assert hasattr(L, name), name
    assert L.upsnet_version(None) == 90
    # lib() binds every declaration, one argtype per parameter (counted here from the raw declaration)
    bound = _lib.lib()
    for name, params in re.findall(r"\bint\s+(upsnet_\w+)\s*\(([^)]*)\)\s*;", re.sub(r"/\*.*?\*/", "", header, flags=re.S)):
        assert len(getattr(bound, name).argtypes) == params.count(",") + 1, name
        assert getattr(bound, name).argtypes == decls[name], name
    vp, i, f, d, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_double, ctypes.c_size_t
    assert decls["upsnet_version"] == [vp]
    assert decls["upsnet_rpn_targets"] == [vp, i, vp, vp, vp, i, i, d, d, d, f, f, i, i, ctypes.c_ulonglong,
                                           vp, vp, vp, vp, vp, vp, sz, vp]
    assert decls["upsnet_roi_align_fpn_forward"] == [vp] * 4 + [i] * 4 + [vp] + [i] * 4 + [vp] * 4
    assert decls["upsnet_cocoeval_workspace_bytes"] == [i, i, ctypes.c_longlong, vp]
    odd = tmp_path / "odd.h"
    odd.write_text("int upsnet_odd(const float *x, short n, void *stream);\n")
    with pytest.raises(_lib.UpsnetError, match="short n"):
        _lib.declarations(str(odd))


def test_ops_fail_loudly_without_cuda_tensors():
    import upsnet_b200
    from upsnet_b200._lib import UpsnetError
    with pytest.raises(UpsnetError):
        upsnet_b200.roi_align(torch.zeros(1, 4, 8, 8), torch.zeros(1, 5), 7, 7, 0.25)
    with pytest.raises(UpsnetError):
        upsnet_b200.conv2d(torch.zeros(1, 4, 8, 8), torch.zeros(4, 4, 3, 3))
