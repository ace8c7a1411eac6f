"""Ground-truth rasteriser, CPU half: the annToRLE restatement (tests/gt_rle_oracle.py) against hand-derived masks, the
h x w toggle formulation the kernel uses against the literal rleFrPoly on seeded random polygons at non-square sizes,
rleMerge's union, the frPyObjects dispatch, and the host packing (ops.pack_segmentations) with its run bound."""
import numpy as np
import pytest

import gt_rle_oracle as GO
from proposal_target_oracle import rle_decode, rle_fr_poly


def decode(R):
    h, w = R['size']
    return rle_decode(np.asarray(R['counts'], np.int64), h, w)


def canonical(c):
    c = np.asarray(c, np.int64)
    return c.size >= 1 and (c[1:] > 0).all()


# ------------------------------------------------------------------------------------------------
# hand-derived masks
# ------------------------------------------------------------------------------------------------
def test_rectangle_and_triangle_by_hand():
    h, w = 9, 13
    m = decode(GO.ann_to_rle([[2, 3, 6, 3, 6, 6, 2, 6]], h, w))
    want = np.zeros((h, w), np.uint8)
    want[3:6, 2:6] = 1                                     # x in [2, 6), y in [3, 6)
    assert np.array_equal(m, want)
    # right triangle (0,0) (8,0) (0,8): column x holds rows 0 .. 6 - x (centres on the hypotenuse are out)
    m = decode(GO.ann_to_rle([[0, 0, 8, 0, 0, 8]], h, w))
    want = np.zeros((h, w), np.uint8)
    for x in range(8):
        want[:7 - x, x] = 1
    assert np.array_equal(m, want)


def test_square_crossing_right_and_bottom_edges():
    # y clamped to h: the lower edge's boundary points land on row 0 of the next column, which the sorted indices of
    # maskApi.c treat as the end of this column's run; the last column's falls off the canvas
    h, w = 6, 8
    R = GO.ann_to_rle([[4, 3, 40, 3, 40, 40, 4, 40]], h, w)
    want = np.zeros((h, w), np.uint8)
    want[3:, 4:] = 1
    assert np.array_equal(decode(R), want)
    assert np.array_equal(GO.toggle_union_rle([[4, 3, 40, 3, 40, 40, 4, 40]], h, w), R['counts'])


def test_disjoint_and_overlapping_parts_unite():
    h, w = 10, 12
    a, b, c = [0, 0, 4, 0, 4, 4, 0, 4], [7, 5, 11, 5, 11, 9, 7, 9], [2, 2, 6, 2, 6, 6, 2, 6]
    want = np.zeros((h, w), np.uint8)
    want[0:4, 0:4] = 1
    want[5:9, 7:11] = 1
    R = GO.ann_to_rle([a, b], h, w)
    assert np.array_equal(decode(R), want) and canonical(R['counts'])
    want = np.zeros((h, w), np.uint8)
    want[0:4, 0:4] = 1
    want[2:6, 2:6] = 1                                     # the union, not the XOR
    R = GO.ann_to_rle([a, c], h, w)
    assert np.array_equal(decode(R), want) and canonical(R['counts'])
    assert np.array_equal(GO.toggle_union_rle([a, c], h, w), R['counts'])


def test_box_list_reading_and_empty_list():
    h, w = 10, 12
    # len(segm[0]) == 4: every entry is a box [x, y, bw, bh] (rleFrBbox), not a 2-vertex polygon
    R = GO.ann_to_rle([[1, 2, 3, 4], [8, 0, 2, 2]], h, w)
    want = np.zeros((h, w), np.uint8)
    want[2:6, 1:4] = 1
    want[0:2, 8:10] = 1
    assert np.array_equal(decode(R), want)
    # later entries of a polygon list with 4 or 2 coordinates are polygons of 2 or 1 vertices: empty masks
    R = GO.ann_to_rle([[1, 2, 5, 2, 5, 6], [0, 0, 9, 9], [3, 3]], h, w)
    assert np.array_equal(decode(R), decode(GO.ann_to_rle([[1, 2, 5, 2, 5, 6]], h, w)))
    with pytest.raises(IndexError):
        GO.ann_to_rle([], h, w)


def test_first_run_may_be_zero_and_full_canvas():
    h, w = 4, 5
    R = GO.ann_to_rle([[-1, -1, 9, -1, 9, 9, -1, 9]], h, w)
    assert list(R['counts']) == [0, h * w]
    R = GO.ann_to_rle([[-1, -1, 9, -1, 9, 9, -1, 9], [1, 1, 2, 1, 2, 2]], h, w)
    assert list(R['counts']) == [0, h * w]


# ------------------------------------------------------------------------------------------------
# the toggle formulation and rleMerge against the literal code
# ------------------------------------------------------------------------------------------------
SIZES = [(480, 640), (640, 427), (7, 300), (1024, 2048)]


@pytest.mark.parametrize("hw", SIZES, ids=["%dx%d" % s for s in SIZES])
def test_toggle_formulation_matches_rle_fr_poly(hw):
    h, w = hw
    rng = np.random.default_rng([h, w])
    n = 300 if h * w > 10 ** 6 else 600
    for i in range(n):
        xy = GO.random_polygon(rng, h, w, i % 6)
        want = np.asarray(rle_fr_poly(xy, h, w), np.uint32)
        got = GO.encode_flat(GO.toggle_flat(xy, h, w))
        assert np.array_equal(got, want), (h, w, i, xy)
        assert canonical(want) and int(want.astype(np.int64).sum()) == h * w


@pytest.mark.parametrize("hw", SIZES[:3], ids=["%dx%d" % s for s in SIZES[:3]])
def test_union_of_parts_matches_rle_merge(hw):
    h, w = hw
    rng = np.random.default_rng([h, w, 1])
    for i in range(150):
        parts = [GO.random_polygon(rng, h, w, int(rng.integers(0, 6))) for _ in range(int(rng.integers(1, 5)))]
        if i % 5 == 0:                                          # 4- and 2-coordinate polygons after the first
            parts += [parts[0][:4], parts[0][:2]]
        R = GO.ann_to_rle(parts, h, w)
        assert np.array_equal(GO.toggle_union_rle(parts, h, w), R['counts']), (h, w, i)
        want = np.zeros((h, w), np.uint8)
        for p in parts:
            want |= rle_decode(np.asarray(rle_fr_poly(p, h, w), np.int64), h, w)
        assert np.array_equal(decode(R), want) and canonical(R['counts'])


def test_rle_merge_intersect_and_size_mismatch():
    rng = np.random.default_rng(3)
    a, b = (rng.random((2, 6, 7)) < 0.5).astype(np.uint8)
    Ra = {'size': [6, 7], 'counts': GO.encode_flat(a.T.reshape(-1))}
    Rb = {'size': [6, 7], 'counts': GO.encode_flat(b.T.reshape(-1))}
    assert np.array_equal(decode(GO.rle_merge([Ra, Rb], 1)), a & b)
    assert np.array_equal(decode(GO.rle_merge([Ra, Rb], 0)), a | b)
    assert GO.rle_merge([Ra, {'size': [7, 6], 'counts': Rb['counts']}])['size'] == [0, 0]


# ------------------------------------------------------------------------------------------------
# the host packing
# ------------------------------------------------------------------------------------------------
def test_pack_segmentations_layout_and_bound():
    from upsnet_b200.operators import pack_segmentations
    h, w = 480, 640
    rng = np.random.default_rng(5)
    segms = []
    for i in range(120):
        if i % 10 == 3:
            segms.append([[float(v) for v in rng.uniform(0, 200, 4)] for _ in range(2)])          # box list
        elif i % 10 == 7:
            m = (rng.random((h, w)) < 0.001).astype(np.uint8)
            segms.append({'size': [h, w], 'counts': GO.encode_flat(m.T.reshape(-1)).tolist()})   # crowd RLE
        else:
            segms.append([GO.random_polygon(rng, h, w, int(rng.integers(0, 6))) for _ in range(int(rng.integers(1, 4)))])
    pk = pack_segmentations(segms, h, w)
    total = 0
    for g, s in enumerate(segms):
        R = GO.ann_to_rle(s, h, w)
        total += len(R['counts'])
        if isinstance(s, dict):
            assert pk.ann_poly[g] == pk.ann_poly[g + 1]
            assert np.array_equal(pk.src_counts[pk.src_off[g]:pk.src_off[g + 1]], R['counts'])
        else:
            assert pk.src_off[g] == pk.src_off[g + 1]
            polys = [pk.verts[2 * pk.poly_vert[q]:2 * pk.poly_vert[q + 1]]
                     for q in range(pk.ann_poly[g], pk.ann_poly[g + 1])]
            assert np.array_equal(GO.toggle_union_rle(polys, h, w), R['counts'])
    assert total <= pk.bound
    assert pk.sizes.shape == (2, len(segms)) and (pk.sizes == [[h], [w]]).all()


def test_pack_segmentations_rejects():
    from upsnet_b200.operators import pack_segmentations
    for bad in ([], [[1, 2, 3]], [[1, 2, 3, 4], [1, 2, 3]], [[0, 0, 1e9, 0, 1e9, 1e9]], [[0, 0, float("nan"), 0, 3, 3]]):
        with pytest.raises(ValueError):
            pack_segmentations([bad], 10, 10)
    # the existing host parser still refuses polygons
    from upsnet_b200.evaluation import gt_rle
    with pytest.raises(ValueError, match="polygon"):
        gt_rle([[0, 0, 4, 0, 4, 4]])


def test_against_pycocotools():
    mask_utils = pytest.importorskip("pycocotools.mask")
    rng = np.random.default_rng(11)
    for h, w in SIZES[:3]:
        for i in range(60):
            segm = [GO.random_polygon(rng, h, w, int(rng.integers(0, 6))) for _ in range(int(rng.integers(1, 4)))]
            if i % 7 == 0:
                segm = [[float(v) for v in rng.uniform(0, 100, 4)]]
            want = mask_utils.decode(mask_utils.merge(mask_utils.frPyObjects(segm, h, w)))
            assert np.array_equal(decode(GO.ann_to_rle(segm, h, w)), want)
