"""The FCN ROI loss oracle (tests/fcn_roi_loss_oracle.py) against what the reference's own FCNHead.forward and loss lines
computed (tests/golden/reference_fcn_roi_loss.npz), and the faults its criteria must reject."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import fcn_roi_loss_oracle as O  # noqa: E402

Z = np.load(os.path.join(HERE, "golden", "reference_fcn_roi_loss.npz"))
LOSS_REL = 1e-5        # the fixture is float32; the oracle float64
GRAD_REL = 1e-4


def fixture(name):
    c = O.case(name)
    assert O.inputs_digest(c) == str(Z["case/%s/inputs_sha256" % name]), "the cases no longer build the fixture's inputs"
    return c


def score_form(c):
    """fcn_score of the case (the score conv of the concat, float64) and its loss / score-conv gradients through the
    commuted form, as the device computes them."""
    feat = O.feat_of(c["levels"])
    w = c["weight"].double().requires_grad_(True)
    b = c["bias"].double().requires_grad_(True)
    return feat, w, b


def agrees(name, loss, dw, db):
    p = "case/%s/" % name
    ok = abs(float(loss) - float(Z[p + "loss"])) <= LOSS_REL * abs(float(Z[p + "loss"]))
    ok &= np.abs(dw.reshape(-1) - Z[p + "d_weight"].reshape(-1)).max() <= GRAD_REL * np.abs(Z[p + "d_weight"]).max()
    ok &= np.abs(db - Z[p + "d_bias"]).max() <= GRAD_REL * np.abs(Z[p + "d_bias"]).max()
    return bool(ok)


def commuted(c, **fault):
    feat, w, b = score_form(c)
    fcn = torch.nn.functional.conv2d(feat, w, b)[0]
    loss = O.loss_from_score(fcn, b, c["rois"], c["seg"], **fault)
    loss.backward()
    return loss.detach(), w.grad.numpy(), b.grad.numpy()


@pytest.mark.parametrize("name", sorted(O.CASES))
def test_oracle_matches_the_reference(name):
    c = fixture(name)
    w = c["weight"].double().requires_grad_(True)
    b = c["bias"].double().requires_grad_(True)
    loss = O.loss_from_feat(c["levels"], w, b, c["rois"], c["seg"])
    loss.backward()
    assert agrees(name, loss.detach(), w.grad.numpy(), b.grad.numpy())


@pytest.mark.parametrize("name", sorted(O.CASES))
def test_commuted_form_matches_the_reference(name):
    assert agrees(name, *commuted(fixture(name)))


def test_cases_cover_the_edges():
    c = O.case("partly_outside")
    _, _, inside = O.roi_align_weights(c["rois"], 16, 24)
    assert float(inside.min()) < 1.0                      # some samples outside the map: the bias correction matters
    c = O.case("thin")
    assert float((c["rois"][:, 3] - c["rois"][:, 1]).min()) * O.SCALE < 1.0
    c = O.case("roi_all_ignored")
    assert bool((c["seg"][1] == 255).all())
    assert all(bool(((O.case(n)["seg"] == 255).float().mean() > 0.1)) for n in O.CASES)
    assert {O.CASES[n][1] for n in O.CASES} == {19, 133} and {O.CASES[n][2] for n in O.CASES} >= {1, 90}


@pytest.mark.parametrize("fault", ["mean_over_valid", "no_bias_correction", "scale_1_8"])
def test_planted_faults_are_rejected(fault):
    kw = {"mean_over_valid": {"mean_over_valid": True}, "no_bias_correction": {"correct_bias": False},
          "scale_1_8": {"scale": 0.125}}[fault]
    names = ["partly_outside", "s133_r90"]
    assert not all(agrees(n, *commuted(fixture(n), **kw)) for n in names)
