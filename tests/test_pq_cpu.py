"""The numpy PQ / label-restore oracle against the reference's own evaluation code (tests/golden/reference_pq.npz, made
by tests/golden/make_reference_pq.py from base_dataset.py and the real cv2.resize)."""
import os

import numpy as np
import pytest

import pq_oracle as P

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_pq.npz"))
CATS = {int(c): {'id': int(c), 'isthing': int(t)} for c, t in zip(GOLD["cat_ids"], GOLD["cat_isthing"])}
CASES = [str(c) for c in GOLD["cases"]]


def case_images(name):
    out = []
    for k in range(int(GOLD[name + "/n"])):
        segs = [{"id": int(r[0]), "category_id": int(r[1]), "iscrowd": int(r[2]), "area": int(r[3])}
                for r in GOLD["%s/%d/segs" % (name, k)]]
        out.append((GOLD["%s/%d/pan" % (name, k)], GOLD["%s/%d/gt" % (name, k)], segs))
    return out


def stat_array(stat):
    a = np.zeros((256, 4))
    for c, v in stat.items():
        a[c] = v
    return a


def check_stat(got, want):
    """tp / fp / fn exactly; IoU sums within 1e-12 * tp (correctly rounded quotients, summation order may differ)."""
    assert np.array_equal(got[:, 1:], want[:, 1:])
    assert (np.abs(got[:, 0] - want[:, 0]) <= 1e-12 * np.maximum(want[:, 1], 1)).all()


def check_summary(summarize, name):
    if int(GOLD[name + "/raises"]):
        with pytest.raises(ZeroDivisionError):
            summarize()
        return
    res = summarize()
    for r, key in enumerate(("All", "Things", "Stuff")):
        want = GOLD[name + "/summary"][r]
        assert res[key]["n"] == int(want[3])
        assert np.allclose([res[key]["pq"], res[key]["sq"], res[key]["rq"]], want[:3], rtol=1e-12, atol=1e-14)
    pc = GOLD[name + "/per_class"]
    assert sorted(res["per_class"]) == sorted(CATS)
    for c, v in res["per_class"].items():
        assert np.allclose([v["pq"], v["sq"], v["rq"]], pc[c], rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize("name", CASES)
def test_oracle_pq_matches_reference(name):
    stat = {}
    for pan, gt, segs in case_images(name):
        P.pq_image(pan, gt, segs, CATS, stat)
    check_stat(stat_array(stat), GOLD[name + "/stat"])
    check_summary(lambda: _summarize(stat), name)


def _summarize(stat):
    res = {}
    for name, isthing in (("All", None), ("Things", True), ("Stuff", False)):
        res[name], pc = P.pq_average(stat, CATS, isthing)
        if name == "All":
            res["per_class"] = pc
    return res


def test_host_pq_average_matches_oracle():
    from upsnet_b200.evaluation import pq_average
    stat = {}
    for pan, gt, segs in case_images("multi_image"):
        P.pq_image(pan, gt, segs, CATS, stat)
    for isthing in (None, True, False):
        assert pq_average(stat, CATS, isthing) == P.pq_average(stat, CATS, isthing)
    with pytest.raises(ZeroDivisionError):
        pq_average({}, CATS, None)


def test_pack_segments_dict_semantics():
    from upsnet_b200.evaluation import pack_segments
    segs = [{"id": 9, "category_id": 1, "iscrowd": 0, "area": 5}, {"id": 3, "category_id": 2, "iscrowd": 1, "area": 7},
            {"id": 9, "category_id": 4, "iscrowd": 1, "area": 8}]
    t = pack_segments(segs)
    assert t.tolist() == [[3, 9], [2, 4], [1, 1], [7, 8], [1, 0]]      # sorted by id; id 9: last entry, first position


def test_oracle_pq_unknown_prediction_category_raises():
    pan, gt, segs = case_images("perfect")[0]
    pan = pan.copy()
    pan[0, 0, 0] = 200
    with pytest.raises(KeyError):
        P.pq_image(pan, gt, segs, CATS)


@pytest.mark.parametrize("k", range(int(GOLD["restore/n"])))
def test_oracle_label_restore_matches_cv2(k):
    Hp, Wp = (int(v) for v in GOLD["restore/%d/shape" % k])
    got = P.label_restore(P.restore_label(Hp, Wp, k), GOLD["restore/%d/im_info" % k])
    assert got.dtype == np.int64 and got.shape == tuple(GOLD["restore/%d/want_shape" % k])
    assert P.digest(got) == str(GOLD["restore/%d/want_sha256" % k])        # bit-exact vs cv2.resize


def test_label_restore_geometry_matches_oracle():
    from upsnet_b200.operators import label_restore_geometry
    for k in range(int(GOLD["restore/n"])):
        info = GOLD["restore/%d/im_info" % k]
        h, w, fx, oh, ow = label_restore_geometry(info)
        assert (oh, ow) == tuple(GOLD["restore/%d/want_shape" % k])
        assert (h, w) == (int(info[0]), int(info[1]))
