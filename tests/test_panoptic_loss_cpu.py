"""The panoptic-loss oracle (tests/panoptic_loss_oracle.py) against what the reference's own modules computed
(tests/golden/reference_panoptic_loss.npz), and the host half of the keep_inds draw."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import panoptic_loss_oracle as PL  # noqa: E402
import rpn_target_oracle as RO  # noqa: E402

Z = np.load(os.path.join(HERE, "golden", "reference_panoptic_loss.npz"))
CASES = sorted(PL.SMALL)


def fixture_case(name):
    """The stored inputs as a case dict.  mask_score is rebuilt with noise in the channels that take no part; fcn_score
    is the seeded generator's, checked against the stored digest."""
    p = name + "/"
    _, S, nc, h, w, G, k, void = PL.SMALL[name]
    fcn = PL.case(PL.SMALL[name])["fcn"]
    assert PL.digest(fcn) == str(Z[p + "fcn_sha256"]), "the generator no longer builds the fcn_score of the fixture"
    cls, sel = Z[p + "cls"], Z[p + "mask_sel"]
    ms = np.random.default_rng(1).standard_normal((len(cls), nc, 28, 28)).astype(np.float32)
    ms[np.arange(len(cls)), cls] = sel
    return dict(fcn=fcn, mask_score=ms, rois=Z[p + "rois"], cls=cls, seg_gt=Z[p + "seg_gt"].astype(np.int64),
                mask_gt=Z[p + "mask_gt"], keep=Z[p + "keep"] if void else None, num_classes=nc, enable_void=void)


def close(got, want, rel):
    return np.abs(got - want).max() <= rel * np.abs(want).max()


@pytest.mark.parametrize("name", CASES)
def test_generator_reproduces_the_stored_inputs(name):
    c, f = PL.case(PL.SMALL[name]), fixture_case(name)
    for key in ("rois", "cls", "seg_gt", "mask_gt"):
        assert np.array_equal(c[key], f[key]), key
    assert np.array_equal(PL.selected(c).numpy(), Z[name + "/mask_sel"])


@pytest.mark.parametrize("name", CASES)
def test_oracle_fp32_matches_the_reference(name):
    p = name + "/"
    got = PL.run(fixture_case(name), torch.float32)
    assert np.array_equal(got["gt"], Z[p + "gt"])
    assert got["correct"] == int(Z[p + "correct"]) and got["ignored"] == int(Z[p + "ignored"])
    assert abs(got["loss"] - float(Z[p + "loss"])) <= 1e-6 * abs(float(Z[p + "loss"]))
    assert abs(got["accuracy"] - float(Z[p + "accuracy"])) <= 1e-6
    ns = got["logits"].shape[1] - Z[p + "logits_inst"].shape[1]
    assert ns == 19 - 9 + 1 or ns == 133 - 81 + 1
    assert np.array_equal(got["logits"][:, :ns], fixture_case(name)["fcn"][:, :ns])     # the stuff channels are fcn_score's
    assert close(got["logits"][:, ns:], Z[p + "logits_inst"], 1e-6)
    # both sides are float32 sums of up to a few hundred terms per element, taken in different orders (matrix products
    # here, ATen's scatter in the fixture): a few float32 ulps of the largest element
    assert close(got["d_fcn"], Z[p + "d_fcn"], 2e-6)
    assert close(got["d_mask"], Z[p + "d_mask"], 2e-6)


def test_cases_hold_what_they_promise():
    c = PL.case(PL.SMALL["cityscapes_void"])
    h, w = c["fcn"].shape[2:]
    b = c["rois"][:, 1:] * np.float32(0.25)
    wid = b[:, 2].astype(np.int64) - b[:, 0].astype(np.int64) + 1
    assert (b[:, 2] > w).any() and (b[:, 3] > h).any()                  # past the right / bottom edge
    assert (wid == 1).any() and (wid > 28).any() and ((wid > 1) & (wid < 28)).any()
    assert (c["cls"] == 0).any() and len(set(c["cls"].tolist())) < len(c["cls"])
    assert (c["mask_gt"] == 255).any() and (c["seg_gt"] == 255).any()
    assert ((c["mask_gt"] == 1).sum(0) > 1).any()                       # overlapping masks: the overwrite order matters
    assert len(c["keep"]) < c["mask_gt"].shape[0] and not np.array_equal(c["keep"], np.sort(c["keep"]))
    gt = PL.panoptic_gt(c["seg_gt"], c["mask_gt"], c["keep"], 19, 9)
    num_stuff, k = 11, len(c["keep"])
    assert ((c["seg_gt"] >= num_stuff) & (c["seg_gt"] < 255) & (gt == num_stuff + k)).any()   # thing label, no mask


def test_draw_keep():
    from upsnet_b200.training import draw_keep, draw_keys
    for G, f in ((1, 0.5), (7, 0.5), (40, 0.9), (300, 0.33), (5, 0.1)):
        d = draw_keep(G, f, seed=3)
        assert d.dtype == np.int64 and len(d) == max(int(G * f), 1) and len(set(d.tolist())) == len(d)
        assert d.min() >= 0 and d.max() < G
        assert np.array_equal(d, draw_keep(G, f, seed=3))
        keys = draw_keys(3, G)
        assert np.array_equal(d, np.argsort(keys, kind="stable")[:len(d)])
    assert not np.array_equal(draw_keep(300, 0.5, seed=3), draw_keep(300, 0.5, seed=4))
    np.random.seed(5)
    a = draw_keep(50, 0.5)
    np.random.seed(5)
    assert np.array_equal(a, draw_keep(50, 0.5))
    # the rule of the target classes (stream 0), and three stored keys of seed 9
    for seed in (0, 9, 2 ** 63 + 11):
        assert np.array_equal(draw_keys(seed, 1000), RO.draw_keys(seed, 1000, 0))
    assert draw_keys(9, 3).tolist() == [12587370737594032228, 309689372594955804, 16731224329868871185]


def test_gt_rois_helper():
    from upsnet_b200.training import gt_rois
    e = dict(boxes=np.array([[1, 2, 30, 40], [5, 6, 70, 80], [9, 9, 20, 20]], np.float32), gt_classes=np.array([3, 0, 2]),
             is_crowd=np.array([0, 0, 1]))
    rois, cls = gt_rois(e, np.float32(1.3), "cpu")
    assert rois.dtype == torch.float32 and cls.dtype == torch.int64
    assert np.array_equal(rois.numpy(), np.hstack((np.zeros((1, 1), np.float32), e["boxes"][:1] * np.float32(1.3))))
    assert cls.tolist() == [3]
