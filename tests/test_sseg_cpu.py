"""The numpy semantic-segmentation oracle and the host-side index tables against the reference's own evaluate_ssegs and
PIL (tests/golden/reference_sseg.npz, made by tests/golden/make_reference_sseg.py)."""
import os

import numpy as np
import pytest

import pq_oracle as P
import sseg_oracle as S

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_sseg.npz"))
CASES = [str(c) for c in GOLD["cases"]]


def case_images(name):
    """[(pred, gt, im_info or None)] of a fixture case."""
    out = []
    for k in range(int(GOLD[name + "/n"])):
        key = "%s/%d/im_info" % (name, k)
        out.append((GOLD["%s/%d/pred" % (name, k)], GOLD["%s/%d/gt" % (name, k)], GOLD[key] if key in GOLD.files else None))
    return out


def check_results(res, matrix, lines):
    """Exact matrix; IU_array / meanIU bit-equal to the reference's formula on it and equal to its logged strings."""
    assert res["confusion_matrix"].dtype == np.float64
    assert np.array_equal(res["confusion_matrix"], matrix)
    tp = np.diag(matrix)
    want_iu = tp / np.maximum(1.0, matrix.sum(1) + matrix.sum(0) - tp)
    assert np.array_equal(res["IU_array"], want_iu)
    assert res["meanIU"] == want_iu.mean()
    assert S.log_lines(res) == [str(s) for s in lines]


@pytest.mark.parametrize("name", CASES)
def test_oracle_sseg_matches_reference(name):
    C = int(GOLD[name + "/C"])
    m = np.zeros((C, C))
    for pred, gt, info in case_images(name):
        m += S.confusion(pred, gt, C, info)
    check_results(S.summarize(m), GOLD[name + "/matrix"], GOLD[name + "/lines"])


def test_oracle_sseg_large_rebuilt_matches_reference():
    pred, gt = S.synthetic_case(0, 1024, 2048, 19)
    check_results(S.summarize(S.confusion(pred, gt, 19)), GOLD["large/matrix"], GOLD["large/lines"])


def test_fixture_covers_the_quirks():
    """The cases exercise what they are named for (so a fixture regenerated with other sizes keeps its meaning)."""
    def first(name):
        return case_images(name)[0]
    assert (first("all_ignored")[1] == 255).all() and not GOLD["all_ignored/matrix"].any()
    gt = first("gt_out_of_range")[1]
    assert ((gt >= 19) & (gt < 255)).mean() > 0.2
    assert (first("pred_aliasing")[0] >= 19).any()
    p = first("int64_wrap")[0]
    assert p.dtype == np.int64 and (p < 0).any() and (p > 255).any()
    assert not GOLD["class_absent/matrix"][7].any() and not GOLD["class_absent/matrix"][:, 7].any()
    assert int(GOLD["five_images/n"]) == 5
    assert str(GOLD["coco_equal/variant"]) == "coco" and int(GOLD["coco_equal/C"]) == 133
    pairs = GOLD["pil/pairs"]
    closed = [not np.array_equal(S.pil_index(a, b), np.floor((np.arange(b) + 0.5) * (a / b)).astype(np.int64)) for a, b in pairs]
    assert sum(closed) >= 10


def test_pil_index_rule_matches_pil_tables():
    from upsnet_b200.evaluation import pil_nearest_index
    pairs = GOLD["pil/pairs"]
    tabs = np.split(GOLD["pil/tables"], np.cumsum(pairs[:, 1])[:-1])
    for (n_in, n_out), want in zip(pairs, tabs):
        assert np.array_equal(S.pil_index(int(n_in), int(n_out)), want), (n_in, n_out)
        assert np.array_equal(pil_nearest_index(int(n_in), int(n_out)), want), (n_in, n_out)


@pytest.mark.parametrize("name", [c for c in CASES if c + "/0/im_info" not in GOLD.files])
def test_index_tables_equal_oracle_resize(name):
    from upsnet_b200.evaluation import sseg_index_tables
    for pred, gt, _ in case_images(name):
        ph, pw = pred.shape[-2:]
        rows, cols = sseg_index_tables((ph, pw), gt.shape)
        assert rows.dtype == np.int32 and cols.dtype == np.int32
        src = np.arange(ph * pw).reshape(ph, pw)
        assert np.array_equal(src[rows][:, cols], S.pil_resize(src, *gt.shape))


def test_index_tables_compose_restore_and_pil():
    """With im_info the tables pick what the cv2 restore followed by Pillow's resize picks, for the fixture's network-
    resolution cases and for gt sizes off the restored size."""
    from upsnet_b200.evaluation import sseg_index_tables
    geoms = [(GOLD[n + "/0/pred"].shape[-2:], GOLD[n + "/0/gt"].shape, GOLD[n + "/0/im_info"]) for n in ("netres", "netres_coco")]
    geoms += [((1024, 2048), (1024, 2048), np.array([1024, 2048, 1.0], np.float32)),
              ((1344, 1344), (427, 640), np.array([800, 1199, 800 / 427], np.float32)),
              ((1344, 1344), (426, 641), np.array([800, 1199, 800 / 427], np.float32))]
    for (Hp, Wp), gt_hw, info in geoms:
        ys = np.broadcast_to(np.arange(Hp)[:, None], (Hp, Wp))
        xs = np.broadcast_to(np.arange(Wp)[None, :], (Hp, Wp))
        # the restore wraps to uint8: carry each source coordinate through it as a low and a high byte
        src_y = P.label_restore(ys % 256, info) + 256 * P.label_restore(ys // 256, info)
        src_x = P.label_restore(xs % 256, info) + 256 * P.label_restore(xs // 256, info)
        rows, cols = sseg_index_tables((Hp, Wp), gt_hw, info)
        assert np.array_equal(rows, S.pil_resize(src_y, *gt_hw)[:, 0])
        assert np.array_equal(cols, S.pil_resize(src_x, *gt_hw)[0])


def test_index_tables_reject_bad_geometry():
    from upsnet_b200.evaluation import sseg_index_tables
    with pytest.raises(ValueError, match="outside"):
        sseg_index_tables((64, 96), (80, 120), np.array([65, 80, 0.8], np.float32))
    with pytest.raises(ValueError, match="outside"):
        sseg_index_tables((64, 96), (80, 120), np.array([50, 97, 0.8], np.float32))


def test_segmentation_iou_rejects_class_counts():
    from upsnet_b200 import SegmentationIoU
    for c in (0, 225):
        with pytest.raises(ValueError):
            SegmentationIoU(c, device="cuda:0")
