"""RPN training targets, CPU half: the numpy restatement (tests/rpn_target_oracle.py) against the reference's executed
add_rpn_blobs (tests/golden/reference_rpn_targets.npz), its IoU against the compiled bbox_overlaps, and the draw rule."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import rpn_target_oracle as RO  # noqa: E402

Z = np.load(os.path.join(HERE, "golden", "reference_rpn_targets.npz"))
CASES = [str(c) for c in Z["cases"]]


def case(name):
    entry = {k: Z["%s/%s" % (name, k)] for k in ("boxes", "gt_classes", "is_crowd")}
    entry["height"], entry["width"] = (int(v) for v in Z[name + "/hw"])
    max_size, straddle = (int(v) for v in Z[name + "/cfg"])
    return entry, float(Z[name + "/scale"]), RO.config(max_size=max_size, straddle=straddle), int(Z[name + "/seed"])


def ulps(a, b):
    ai = a.view(np.int32).astype(np.int64)
    bi = b.view(np.int32).astype(np.int64)
    ai = np.where(ai < 0, -(ai & 0x7FFFFFFF), ai)
    bi = np.where(bi < 0, -(bi & 0x7FFFFFFF), bi)
    return np.abs(ai - bi)


def check_against_fixture(name, got):
    _, _, cfg, _ = case(name)
    for k in ("labels", "inside", "outside"):
        assert np.array_equal(got[k], Z["%s/%s" % (name, k)]), (name, k)
    xy = RO.xy_mask(cfg)
    want_t = Z[name + "/targets"]
    assert np.array_equal(got["targets"][xy], want_t[xy]), name
    assert ulps(got["targets"][~xy], want_t[~xy]).max() <= 4, name


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference(name):
    entry, scale, cfg, seed = case(name)
    got = RO.from_roidb(entry, scale, cfg, seed)
    check_against_fixture(name, got)
    log = [(k, n, s) for k, n, s in zip(Z[name + "/log_kind"], Z[name + "/log_n"], Z[name + "/log_size"])]
    assert [(kind == "array", n, s) for kind, n, s in got["log"]] == log


# the quirk each fixture exists for
QUIRKS = {"fg_subsample": "fg_subsampled", "no_negatives": "no_negatives", "zero_max_box": "zero_max_box",
          "ties": "tied_max", "relabelled": "relabelled", "iou_exact": ("pos_exact", "neg_exact"),
          "g1500": "fg_subsampled"}


@pytest.mark.parametrize("name", sorted(QUIRKS))
def test_fixture_reaches_its_quirk(name):
    flags = QUIRKS[name] if isinstance(QUIRKS[name], tuple) else (QUIRKS[name],)
    for f in flags:
        assert int(Z["%s/flag/%s" % (name, f)]) == 1, (name, f)
    assert int(Z["g1500/boxes"].shape[0]) > 1024        # more than one shared-memory chunk of boxes


def test_straddle_and_filter_cases():
    assert [int(v) for v in Z["straddle_all/cfg"]][1] == -1 and [int(v) for v in Z["straddle_16/cfg"]][1] == 16
    e, _, _, _ = case("crowd_filtered")
    assert (e["is_crowd"] == 1).any() and (e["gt_classes"] == 0).any()
    assert int(Z["g1/boxes"].shape[0]) == 1


def test_oracle_iou_is_the_compiled_bbox_overlaps():
    a, q, want = Z["iou/boxes"], Z["iou/query"], Z["iou/overlaps"]
    got = RO.iou(a, q)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert (want > 0).mean() > 0.02


def test_cython_expression_recorded():
    assert str(Z["cython_version"]).startswith("3.")
    assert str(Z["c_stmt/iw"]).endswith("+ 1.0)")
    assert str(Z["c_stmt/ua"]).startswith("((double)")


@pytest.mark.parametrize("name", [c[0] for c in RO.FULL])
def test_full_size_digest(name):
    entry, scale, cfg = RO.full_case(name, 0)
    got = RO.from_roidb(entry, scale, cfg, int(Z["full/seed"]))
    assert RO.digest(got, cfg) == str(Z["full/%s/sha256" % name])
    assert [n for _, n, _ in got["log"]] == list(Z["full/%s/log_n" % name])


def test_draw_rule_is_uniform():
    """Over 20,000 seeds every position of a 12-candidate list is among the 4 drawn at rate 1/3 (chi-square, 11 dof)."""
    n, size, seeds = 12, 4, 20000
    hits = np.zeros(n)
    for s in range(seeds):
        hits[RO.choice_positions(s * 7919 + 1, n, size, s & 1)] += 1
    expect = seeds * size / n
    chi2 = (((hits - expect) ** 2) / expect).sum()
    assert chi2 < 31.3          # the 0.999 quantile of chi-square with 11 degrees of freedom
    assert len(set(RO.draw_keys(3, 100000, 0).tolist())) == 100000
