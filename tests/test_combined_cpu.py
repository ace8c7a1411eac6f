"""The numpy combined-panoptic oracle (tests/combined_oracle.py) against the reference's own get_combined_pan_result /
_merge_pred_single_core (tests/golden/reference_combined.npz, made by tests/golden/make_reference_combined.py), the
quirks it pins, and the host parsing of the drop-in operators.get_combined_pan_result."""
import os

import numpy as np
import pytest

import combined_oracle as CO
from oracle import oracle as O
from upsnet_b200 import operators as ops

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_combined.npz"))
CASES = [str(c) for c in GOLD["cases"]]


def case(name):
    """(sem, scores, cls, runs, (num_seg_classes, num_classes, score_threshold, fraction_threshold, stuff_area_limit))"""
    runs, off = GOLD[name + "/runs"], GOLD[name + "/run_off"]
    p = GOLD[name + "/params"]
    params = (int(p[0]), int(p[1]), float(p[2]), float(p[3]), int(p[4]))
    return (GOLD[name + "/sem"], GOLD[name + "/scores"], GOLD[name + "/cls"],
            [runs[off[d]:off[d + 1]] for d in range(len(off) - 1)], params)


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference(name):
    sem, scores, cls, runs, params = case(name)
    if not int(GOLD[name + "/order_ok"]):
        pytest.skip("the executed argsort did not give the stable order on these exact ties (the reference leaves it open)")
    assert np.array_equal(CO.combined_pan_result(sem, scores, cls, runs, *params), GOLD[name + "/pan"])


def test_fixture_covers_the_tie_rule():
    """At least the hand-made tie cases were ordered by the rule by the executed argsort, so the rule is pinned."""
    assert int(GOLD["ties_within_class/order_ok"]) and int(GOLD["ties_across_classes/order_ok"])


def test_oracle_large_image_digest():
    sem, scores, cls, runs = CO.large_case()
    p = GOLD["large/params"]
    pan = CO.combined_pan_result(sem, scores, cls, runs, int(p[0]), int(p[1]), float(p[2]), float(p[3]), int(p[4]))
    assert int(GOLD["large/order_ok"]) == 1
    assert CO.digest(pan) == str(GOLD["large/sha256"])
    assert int((pan[..., 1] > 0).sum()) == int(GOLD["large/instances"])


def instances(name):
    pan = GOLD[name + "/pan"]
    return sorted({(int(a), int(b)) for a, b in pan[pan[..., 1] > 0][:, :2]})


def test_reference_quirks():
    # score exactly float32(0.6) is kept, the float below it is not (class 2 -> 12, class 4 -> 14)
    assert instances("score_at_threshold") == [(12, 1)]
    # 7 of 10 pixels free: float32(0.7) is not < float32(0.7), kept (numpy 1's float64 compare would drop it)
    assert np.float32(7) / np.float32(10) == np.float32(0.7) and float(np.float32(0.7)) < 0.7
    assert instances("fraction_7_of_10") == [(11, 1), (12, 1)]
    assert instances("fraction_69_of_100") == [(11, 1)]
    assert instances("none_above_threshold") == [] and instances("no_detections") == []
    # the 256th instance of a class writes 0: its cell stays free and a later detection of class 4 claims it
    pan = GOLD["wrap_256/pan"]
    assert int((pan[..., 1] > 0).sum()) == 4 * 299 + 4
    assert (pan[..., 0] == 14).sum() == 4
    # stuff area: 64 pixels (= limit) stay, 63 become void
    pan = GOLD["stuff_limit/pan"]
    assert (pan[..., 0] == 0).sum() == 64 and (pan[..., 0] == 1).sum() == 0


def test_merge_order_is_stable_argsort_of_the_concatenation():
    rng = np.random.default_rng(5)
    for _ in range(20):
        n = int(rng.integers(0, 60))
        scores = np.round(rng.uniform(0, 1, n), 1).astype(np.float32)
        cls = rng.integers(0, 12, n)
        got = CO.merge_order(scores, cls, 9)
        cat = [d for j in range(1, 9) for d in np.flatnonzero(cls == j)]            # im_post's per-class lists
        want = [cat[k] for k in np.argsort(scores[cat], kind="stable")[::-1]] if cat else []
        assert got == want


def test_dropin_host_parsing():
    rng = np.random.default_rng(11)
    H, W = 30, 41
    scores, cls, runs = CO.random_detections(rng, H, W, 12, 5)
    boxes = [[np.zeros((0, 5), np.float32)]] + [[None] for _ in range(1, 5)]
    masks = [[[]]] + [[None] for _ in range(1, 5)]
    for j in range(1, 5):
        sel = np.flatnonzero(cls == j)
        b = rng.uniform(0, 30, (sel.size, 5)).astype(np.float32)
        b[:, 4] = scores[sel]
        boxes[j][0] = b
        # compressed strings (str and bytes) and one uncompressed list
        masks[j][0] = [{"size": [H, W], "counts": O.rle_to_string(runs[d]).decode() if k % 2 else O.rle_to_string(runs[d])}
                       for k, d in enumerate(sel)]
        if sel.size:
            masks[j][0][0] = {"size": [H, W], "counts": [int(v) for v in runs[sel[0]]]}
    sc, cl, cn, rl = ops.combined_inputs(boxes, masks, 0, H, W)
    order = [d for j in range(1, 5) for d in np.flatnonzero(cls == j)]
    assert np.array_equal(sc, scores[order]) and np.array_equal(cl, cls[order])
    for k, d in enumerate(order):
        assert np.array_equal(cn[k, :rl[k]], runs[d])
    masks[1][0][0] = {"size": [H + 1, W], "counts": masks[1][0][0]["counts"]}
    if len(masks[1][0]):
        with pytest.raises(ValueError):
            ops.combined_inputs(boxes, masks, 0, H, W)
