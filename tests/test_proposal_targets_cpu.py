"""Proposal targets, CPU half: the rleFrPoly restatement against hand-derived masks, the toggle formulation the kernel
uses against it, and the numpy restatement (tests/proposal_target_oracle.py) against the reference's executed
ProposalMaskTarget (tests/golden/reference_proposal_targets.npz)."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import proposal_target_oracle as PO  # noqa: E402
from test_rpn_targets_cpu import ulps  # noqa: E402

Z = np.load(os.path.join(HERE, "golden", "reference_proposal_targets.npz"))
CASES = [str(c) for c in Z["cases"]]


def case(name):
    """-> rois, entry, im_scale, cfg, seed of a fixture case."""
    e = {k: Z["%s/%s" % (name, k)] for k in ("boxes", "gt_classes", "is_crowd", "box_to_gt_ind_map", "gt_overlaps")}
    oo, po, v = Z[name + "/obj_off"], Z[name + "/poly_off"], Z[name + "/verts"]
    segms = []
    for i in range(len(oo) - 1):
        if oo[i + 1] == oo[i]:
            segms.append({"size": [1, 1], "counts": "crowd"})
        else:
            segms.append([v[2 * po[j]:2 * po[j + 1]].tolist() for j in range(oo[i], oo[i + 1])])
    e["segms"] = segms
    K, B, M = (int(x) for x in Z[name + "/cfg"])
    fgf, fgt, bgh, bgl = (float(x) for x in Z[name + "/cfg_f"])
    cfg = PO.config(num_classes=K, batch_rois=B, M=M, fg_fraction=fgf, fg_thresh=fgt, bg_hi=bgh, bg_lo=bgl)
    return Z[name + "/rois_in"], e, np.float32(Z[name + "/scale"]), cfg, int(Z[name + "/seed"])


def check_outputs(got, want, name=""):
    for k in PO.NAMES:
        assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, (name, k, got[k].shape, want[k].shape)
        if k == "bbox_targets":
            xy = PO.dxdy_mask(want[k])
            assert np.array_equal(got[k][xy], want[k][xy]), (name, k)
            assert ulps(got[k][~xy], want[k][~xy]).max(initial=0) <= 4, (name, k)
        else:
            assert np.array_equal(got[k], want[k]), (name, k)


def fixture(name):
    return {k: Z["%s/%s" % (name, k)] for k in PO.NAMES}


def oracle_out(name):
    rois, e, s, cfg, seed = case(name)
    o = PO.proposal_targets(rois, e, s, cfg, seed)
    # the module's dtypes: labels / nongt int64, roi_has_mask uint8, everything else float32
    return o


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference(name):
    check_outputs(oracle_out(name), fixture(name), name)
    log = Z[name + "/log"]
    assert all(s in (0, 1) for s in log[:, 0])


def test_cases_reach_their_rules():
    f = fixture
    assert (f("fg_on_crowd")["labels"] == 5).any()                         # the crowd's class on an fg proposal
    assert len(f("no_fg_fallback")["mask_rois"]) == 1 and (f("no_fg_fallback")["mask_int32"] == -1).all()
    assert f("no_fg_fallback")["roi_has_mask"][0] == 1 and f("no_fg_fallback")["labels"][0] == 0
    assert (f("iou_exact")["labels"] > 0).sum() == 2                       # IoU == fg_thresh is fg
    assert list(f("batch_rows")["nongt_inds"]) == sorted(f("batch_rows")["nongt_inds"])
    fe = f("few_fg_few_bg")
    assert (fe["labels"] > 0).sum() < 8 and len(fe["labels"]) < 32
    # the 1-px roi is fg and its mask is not empty
    m = f("far_outside_1px")["mask_int32"]
    assert (m == 1).any()


def test_full_size_digests():
    for name, *_ in PO.FULL:
        e, rois, scale, cfg = PO.full_case(name, 0)
        got = PO.proposal_targets(rois, e, scale, cfg, int(Z["full/seed"]))
        assert PO.digest(got) == str(Z["full/%s/sha256" % name]), name


# ------------------------------------------------------------------------------------------------
# the rasteriser
# ------------------------------------------------------------------------------------------------
def _rect_expected(x1, y1, x2, y2, M):
    """rleFrPoly of an axis-aligned rectangle with corners (pixel units): columns n with x1 <= n + .5 - .1 ... derived
    from the rule: x boundary points survive at u = 5n + 2 between the vertical edges, y = ceil((5 y + .5) / 5 - .5)."""
    m = np.zeros((M, M), np.uint8)
    X1, X2 = int(5 * x1 + .5), int(5 * x2 + .5)
    Y1, Y2 = int(5 * y1 + .5), int(5 * y2 + .5)
    ya = int(np.ceil(min(max((Y1 + .5) / 5 - .5, 0), M)))
    yb = int(np.ceil(min(max((Y2 + .5) / 5 - .5, 0), M)))
    for n in range(M):
        if X1 <= 5 * n + 2 and 5 * n + 3 <= X2:
            m[ya:yb, n] = 1
    return m


@pytest.mark.parametrize("rect", [(2, 3, 10, 12), (0, 0, 28, 28), (5.3, 7.7, 20.1, 9.9), (-4, -3, 6, 40)])
def test_rectangles_by_hand(rect):
    x1, y1, x2, y2 = rect
    poly = [x1, y1, x2, y1, x2, y2, x1, y2]
    want = _rect_expected(x1, y1, x2, y2, 28)
    assert np.array_equal(PO.rle_mask(poly, 28), want)
    assert np.array_equal(PO.toggle_mask(poly, 28), want)


def test_rectangle_simple_values():
    # a 4 x 3 block at columns 2..5, rows 3..5 of an 8 x 8 mask: x in [2, 6), y in [3, 6)
    m = PO.rle_mask([2, 3, 6, 3, 6, 6, 2, 6], 8)
    want = np.zeros((8, 8), np.uint8)
    want[3:6, 2:6] = 1
    assert np.array_equal(m, want)


def test_triangle_by_hand():
    # right triangle (0,0) (8,0) (0,8) at M = 8: column x's boundary point sits at u = 5x + 2 on the hypotenuse, where
    # v = 40 - (5x + 3) rounds to y = ceil((37 - 5x + .5) / 5 - .5) = 7 - x: rows 0 .. 6 - x, the pixels whose centre
    # (x + .5, y + .5) lies strictly inside (the centres on the hypotenuse are out)
    m = PO.rle_mask([0, 0, 8, 0, 0, 8], 8)
    want = np.zeros((8, 8), np.uint8)
    for x in range(8):
        want[:7 - x, x] = 1
    assert np.array_equal(m, want)
    assert np.array_equal(PO.toggle_mask([0, 0, 8, 0, 0, 8], 8), want)


def test_polygon_crossing_the_edge_and_overlap_union():
    # a square that sticks out of the right and bottom edges: clipped at M (y clamp spills into the next column)
    a = PO.rle_mask([4, 4, 40, 4, 40, 40, 4, 40], 8)
    want = np.zeros((8, 8), np.uint8)
    want[4:, 4:] = 1
    assert np.array_equal(a, want)
    # two overlapping squares: the union, as polys_to_mask_wrt_box sums the decoded masks and thresholds at 0
    box = np.array([0, 0, 8, 8], np.float32)
    u = PO.poly_mask([[0, 0, 5, 0, 5, 5, 0, 5], [3, 3, 7, 3, 7, 7, 3, 7]], box, 8)
    want = np.zeros((8, 8), np.uint8)
    want[0:5, 0:5] = 1
    want[3:7, 3:7] = 1
    assert np.array_equal(u, want)


@pytest.mark.parametrize("seed", range(6))
def test_toggle_formulation_matches_rle_fr_poly(seed):
    """Random polygons, many with vertices outside [0, M] (negative ones included), some steep, some on the .5
    boundary: the edge-by-edge toggles give the literal rleFrPoly mask."""
    rng = np.random.default_rng(seed)
    for M in (28, 7, 32):
        for _ in range(60):
            k = int(rng.integers(3, 12))
            scale = [1.0, 3.0, 40.0][int(rng.integers(0, 3))]
            xy = (rng.uniform(-0.5, 1.5, 2 * k) * M * (scale if rng.random() < 0.2 else 1.0))
            if rng.random() < 0.3:
                xy = np.round(xy * 5) / 5 + 0.1                      # near 5 * c + .5 = integer
            xy = xy.astype(np.float32).astype(np.float64)
            assert np.array_equal(PO.toggle_mask(xy, M), PO.rle_mask(xy, M)), (seed, M, xy.tolist())


def test_generator_is_deterministic_by_construction():
    # the fixtures carry no timestamps: the zip members are written with a fixed date
    import zipfile
    with zipfile.ZipFile(os.path.join(HERE, "golden", "reference_proposal_targets.npz")) as z:
        assert {i.date_time for i in z.infolist()} == {(1980, 1, 1, 0, 0, 0)}
