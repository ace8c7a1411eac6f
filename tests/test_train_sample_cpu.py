"""CPU checks of TrainingSample's host half against what the reference's loader and collate made of each fixture case
(tests/golden/reference_train_sample.npz): the scale draw and the max_size rule, the collated keys / shapes / dtypes
that the GPU test holds the device sample to, and the flip of a roidb entry the GPU training step uses."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import train_sample_cases as TS  # noqa: E402

CASES = TS.load_cases()
IDS = [c["name"] for c in CASES]


def sampler(dataset):
    from upsnet_b200.training import TrainingSample
    return TrainingSample(dataset=dataset, pixel_means=TS.PIXEL_MEANS, **TS.CONFIGS[dataset])


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_scale_draw_matches_reference(case):
    """Same np.random seed: the same scale index and the same im_scale bits as get_image_blob / prep_im_for_blob."""
    np.random.seed(case["np_seed"])
    ind, s = sampler(case["dataset"]).draw_scale(*case["shape"])
    assert ind == case["scale_index"]
    assert np.float64(s).tobytes() == case["im_scale"].tobytes()
    assert type(s) is float


def test_max_size_rule():
    """The cap compares np.round(scale * longest side) with max_size: equal is not capped, one above is."""
    ts = sampler("coco")
    assert ts.im_scale(640, 480, 1000) == 640 / 480.0            # round(1333.33) = 1333: not above 1333
    assert ts.im_scale(672, 480, 1000) == 1333 / 1000.0          # round(1400) > 1333: capped
    assert ts.im_scale(800, 1000, 480) == 1333 / 1000.0          # portrait: the same rule on the height
    assert ts.im_scale(800, 600, 999) == 800 / 600.0             # round(1332) <= 1333


def expected_layout(case):
    """collate's output for the case, from its resized size: the blob padded to 32 (rpn_feat_stride[-2]), the label
    maps at the blob's and a quarter of its padded size, one mask_gt / gt_classes row per drawn roidb row (all rows for
    Cityscapes, the non-crowd rows for COCO), one seg_roi_gt row per non-crowd box of a class > 0 (COCO)."""
    ho, wo = (int(v) for v in case["im_info"][0, :2])
    Hp, Wp = -(-ho // 32) * 32, -(-wo // 32) * 32
    e = case["entry"]
    rows = len(e["gt_classes"]) if case["dataset"] == "cityscapes" else int((e["is_crowd"] == 0).sum())
    data = ["data|tensor|float32|1,3,%d,%d" % (Hp, Wp), "data_4x|tensor|float32|1,3,%d,%d" % (Hp // 4, Wp // 4),
            "im_info|ndarray|float32|1,3"]
    label = ["gt_classes|tensor|%s|%d" % (e["gt_classes"].dtype, rows),
             "mask_gt|tensor|int64|%d,%d,%d" % (rows, Hp // 4, Wp // 4),
             "roidb|dict|%s|" % ",".join(sorted(k for k in TS.ROIDB_KEYS if k in e)),
             "seg_gt|tensor|int64|1,%d,%d" % (Hp, Wp), "seg_gt_4x|tensor|int64|1,%d,%d" % (Hp // 4, Wp // 4)]
    if TS.CONFIGS[case["dataset"]]["with_roi"]:
        n = int(((e["gt_classes"] > 0) & (e["is_crowd"] == 0)).sum())
        label.append("seg_roi_gt|tensor|int64|%d,28,28" % n)
    return data, label


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_collate_layout(case):
    data, label = expected_layout(case)
    assert case["data_layout"] == data
    assert case["label_layout"] == label
    h, w = case["shape"]
    s = float(case["im_scale"])
    assert case["im_info"].dtype == np.float32 and case["im_info"].tolist() == \
        np.array([[np.round(h * s), np.round(w * s), s]], np.float32).tolist()


@pytest.mark.parametrize("case", [c for c in CASES if c["entry"]["flipped"]], ids=[c["name"] for c in CASES
                                                                                  if c["entry"]["flipped"]])
def test_flip_entry_matches_reference(case):
    """TS.flip_entry (used to flip synthetic entries on the GPU) is extend_with_flipped_entries, bit for bit."""
    got = TS.flip_entry(case["base"])
    want = case["entry"]
    assert got["flipped"] and got["boxes"].dtype == want["boxes"].dtype
    assert np.array_equal(got["boxes"].view(np.uint32), want["boxes"].view(np.uint32))
    assert [[np.asarray(p).tobytes() for p in s] for s in got["segms"]] == \
        [[np.asarray(p).tobytes() for p in s] for s in want["segms"]]
