"""The training-loss oracle (tests/train_loss_oracle.py) against what the reference's own RPNLoss, MaskRCNNLoss and
semantic-loss lines computed (tests/golden/reference_train_losses.npz)."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import train_loss_oracle as TL  # noqa: E402

Z = np.load(os.path.join(HERE, "golden", "reference_train_losses.npz"))


def sem_fixture(name):
    seed, S, h, w, pad, ign, _ = TL.SEM_SMALL[name]
    c = TL.semantic_case(seed, S, h, w, pad, ign)
    assert TL.digest(c["fcn"]) + TL.digest(c["seg_gt"]) == str(Z["sem/%s/inputs_sha256" % name]), \
        "the generator no longer builds the inputs of the fixture"
    return c


def rpn_fixture(name):
    c = TL.rpn_case(*TL.RPN_SMALL[name])
    d = "".join(TL.digest(a) for a in c["scores"] + c["preds"]) + "".join(TL.digest(c["label"][k]) for k in sorted(c["label"]))
    assert d == str(Z["rpn/%s/inputs_sha256" % name]), "the generator no longer builds the inputs of the fixture"
    return c


def mrcnn_fixture(name):
    c = TL.mask_rcnn_case(*TL.MRCNN_SMALL[name])
    assert "".join(TL.digest(c[k]) for k in TL.NAMES) == str(Z["mrcnn/%s/inputs_sha256" % name]), \
        "the generator no longer builds the inputs of the fixture"
    return c


def close(got, want, rel):
    return np.abs(got - want).max() <= rel * np.abs(want).max()


def rel(got, want):
    return abs(got - float(want)) / max(abs(float(want)), 1e-30)


@pytest.mark.parametrize("name", sorted(TL.SEM_SMALL))
def test_semantic_oracle_matches_the_reference(name):
    p = "sem/%s/" % name
    got = TL.semantic(sem_fixture(name))
    assert got["n"] == int(Z[p + "n"]) and got["invalid"] == 0
    assert rel(got["loss"], Z[p + "loss"]) <= 1e-6
    assert close(got["d_fcn"], Z[p + "d_fcn"], 1e-6)


@pytest.mark.parametrize("name", sorted(TL.RPN_SMALL))
def test_rpn_oracle_matches_the_reference(name):
    p = "rpn/%s/" % name
    got = TL.rpn(rpn_fixture(name), 256)
    assert rel(got["cls_loss"], Z[p + "cls_loss"]) <= 1e-6 and rel(got["bbox_loss"], Z[p + "bbox_loss"]) <= 1e-6
    for s, ds, dp in zip(TL.STRIDES, got["d_scores"], got["d_preds"]):
        assert close(ds, Z[p + "d_score%d" % s], 1e-6) and close(dp, Z[p + "d_pred%d" % s], 1e-6)


@pytest.mark.parametrize("name", sorted(TL.MRCNN_SMALL))
def test_mask_rcnn_oracle_matches_the_reference(name):
    p = "mrcnn/%s/" % name
    got = TL.mask_rcnn(mrcnn_fixture(name))
    for k in ("cls_loss", "bbox_loss", "mask_loss"):
        assert abs(got[k] - float(Z[p + k])) <= 1e-6 * max(abs(float(Z[p + k])), 1e-30), k
    assert np.float32(got["accuracy"]) == Z[p + "accuracy"]
    for k in ("d_cls", "d_bbox", "d_mask"):
        want = Z[p + k]
        assert np.abs(got[k] - want).max() <= 1e-6 * max(np.abs(want).max(), 1e-30), k


def test_cases_hold_what_they_promise():
    c = TL.semantic_case(*TL.SEM_SMALL["cityscapes"][:6])
    assert (c["seg_gt"][:, -6:] == 255).all() and (c["seg_gt"][:, :, -10:] == 255).all()
    r = TL.rpn_case(*TL.RPN_SMALL["fields_larger"])
    for x, s in zip(r["scores"], TL.STRIDES):
        f = r["label"]["rpn_labels_fpn%d" % s]
        assert f.shape[2] >= x.shape[2] and f.shape[3] >= x.shape[3]         # the reference slices the fields
        if s == 4:                                                           # labels outside the map must not count
            assert f.shape[2] > x.shape[2] and (f[:, :, x.shape[2]:] != -1).any()
    m = TL.mask_rcnn_case(*TL.MRCNN_SMALL["ignored_rows"])
    assert (m["cls_label"] == -1).any() and TL.mask_rcnn(m)["accuracy"] < 0        # the accuracy quirk shows
    assert (TL.mask_rcnn_case(*TL.MRCNN_SMALL["no_mask_target"])["mask_target"] == -1).all()
    assert (Z["mrcnn/no_mask_target/d_mask"] == 0).all() and float(Z["mrcnn/no_mask_target/mask_loss"]) == 0


def test_invalid_labels_are_counted_apart():
    c = TL.semantic_case(11, 5, 6, 8, invalid=0.2)
    got = TL.semantic(c)
    seg = c["seg_gt"]
    assert got["invalid"] == int(((seg != 255) & (seg >= 5)).sum()) > 0
    assert got["n"] == int((seg < 5).sum())
