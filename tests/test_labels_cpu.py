"""CPU checks of the panoptic training labels: the numpy oracle (tests/label_oracle.py) against what the reference's
loaders and collate computed (tests/golden/reference_labels.npz), its Pillow polygon fill against the real Pillow, its
nearest-neighbour tables against the real cv2, and PanopticLabels' host-built tables against the oracle."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import label_oracle as LO  # noqa: E402

GOLD = os.path.join(HERE, "golden", "reference_labels.npz")


def load_cases():
    z = np.load(GOLD)
    out = []
    for name in z["cases"]:
        p = str(name) + "/"
        coords, pc, op = z[p + "coords"], z[p + "poly_coord"], z[p + "obj_poly"]
        polys = [[float(v) for v in coords[pc[i]:pc[i + 1]]] for i in range(len(pc) - 1)]
        segms = [polys[op[g]:op[g + 1]] for g in range(len(op) - 1)]
        entry = dict(boxes=z[p + "boxes"], gt_classes=z[p + "gt_classes"], is_crowd=z[p + "is_crowd"], segms=segms,
                     flipped=bool(z[p + "flipped"]))
        Hb, Wb, with_roi, raises = (int(v) for v in z[p + "meta"])
        ref = {k[len(p) + 4:]: z[k].astype(np.int64) for k in z.files if k.startswith(p + "out_")}
        out.append(dict(name=str(name), entry=entry, label_map=z[p + "label_map"], im_shape=(Hb, Wb),
                        scale=float(z[p + "scale"]), dataset=str(z[p + "dataset"]), with_roi=bool(with_roi),
                        raises=bool(raises), ref=ref))
    return out


CASES = load_cases()


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_oracle_matches_reference(case):
    args = (case["entry"], case["label_map"], case["im_shape"], case["scale"], case["dataset"], case["with_roi"])
    if case["raises"]:
        with pytest.raises(ValueError):
            LO.labels(*args)
        return
    out = LO.labels(*args)
    assert sorted(out) == sorted(case["ref"])
    for k, v in case["ref"].items():
        assert out[k].dtype == np.int64 and out[k].shape == v.shape, k
        np.testing.assert_array_equal(out[k], v, err_msg=k)


@pytest.mark.parametrize("name", ["cityscapes_g50", "coco_g15"])
def test_oracle_full_size_digest(name):
    z = np.load(GOLD)
    entry, lab, im_shape, scale, dataset = LO.full_case(name)
    assert LO.digest(LO.labels(entry, lab, im_shape, scale, dataset, True)) == str(z["full/" + name])


def random_polygon(rng, kind, W, H):
    n = int(rng.integers(3, 9))
    if kind == 0:                       # star-shaped (convex when the radii agree)
        ang = np.sort(rng.random(n) * 2 * np.pi)
        r = 2 + rng.random(n) * 12 * (1 if rng.random() < 0.7 else 0) + rng.random() * 6
        xs, ys = W / 2 + r * np.cos(ang), H / 2 + r * np.sin(ang)
    elif kind == 1:                     # self-intersecting, fractional, partly outside the canvas
        xs, ys = rng.random(n) * (W + 12) - 6, rng.random(n) * (H + 12) - 6
    elif kind == 2:                     # integer vertices: horizontal / vertical edges, repeated and collinear points
        xs, ys = rng.integers(-3, W + 3, n).astype(float), rng.integers(-3, H + 3, n).astype(float)
        if n > 3:
            xs[1], ys[1] = xs[0], ys[0]
            xs[2], ys[2] = (xs[0] + xs[3]) / 2, (ys[0] + ys[3]) / 2
    else:                               # negative coordinates near zero, tiny and far out-of-canvas shapes
        c = rng.uniform(-4, 4, 2)
        s = rng.choice([0.4, 3.0, 30.0])
        xs, ys = c[0] + rng.uniform(-s, s, n), c[1] + rng.uniform(-s, s, n)
    xy = np.empty(2 * n)
    xy[0::2], xy[1::2] = xs, ys
    return [float(v) for v in xy]


def test_pillow_fill_matches_pillow():
    Image = pytest.importorskip("PIL.Image")
    ImageDraw = pytest.importorskip("PIL.ImageDraw")
    rng = np.random.default_rng(2024)
    W, H = 30, 26
    n = 0
    for t in range(16000):
        polys = [random_polygon(rng, t % 4, W, H)]
        if t % 5 == 0:                                  # an instance of several polygons
            polys += [random_polygon(rng, (t // 5) % 4, W, H) for _ in range(int(rng.integers(1, 4)))]
        n += len(polys)
        img = Image.new("L", (W, H), 0)
        canvas = np.zeros((H, W), np.uint8)
        for p in polys:
            ImageDraw.Draw(img).polygon(tuple(p), outline=1, fill=1)
            LO.pillow_fill(canvas, p)
        got = np.array(img)
        if not np.array_equal(got, canvas):
            bad = np.argwhere(got != canvas)
            pytest.fail("polygons %r: Pillow and the restatement differ at (row, col) %s" % (polys, bad.tolist()))
    assert n >= 20000


def test_pillow_fill_hand_cases():
    c = LO.pillow_fill(np.zeros((6, 8), np.uint8), [2.9, 1.2, 2.2, 1.9, 2.5, 1.7])        # one truncated pixel
    assert c.sum() == 1 and c[1, 2] == 1
    c = LO.pillow_fill(np.zeros((6, 8), np.uint8), [-0.5, 1.0, 3.0, 1.0, 3.0, 3.0])       # int(-0.5) = 0, not -1
    assert c[1, 0] == 1 and c[1, 0:4].all()


def test_nearest_tables_match_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(7)
    pairs = 0
    scales = [1.0, 0.5, 0.25, 1.25, 800 / 480.0, 1333 / 640.0, 0.7, 1 / 3.0, 2.0, 600 / 1024.0]
    for n in [1, 2, 3, 7, 31, 45, 61, 87, 100, 255, 480, 513, 640]:
        for s in scales:
            if np.rint(n * s) < 1:
                continue
            a = rng.integers(0, 256, (n, 3)).astype(np.uint8)
            got = cv2.resize(a, None, None, fx=1.0, fy=s, interpolation=cv2.INTER_NEAREST)
            np.testing.assert_array_equal(got, a[LO.nearest_fx(n, s)], err_msg="n=%d fx=%r" % (n, s))
            pairs += 1
    for n in list(range(1, 130)) + [211, 333, 600, 1023]:          # the 28 x 28 seg_roi_gt resize: dsize, not fx
        a = rng.integers(0, 256, (n, 2)).astype(np.uint8)
        got = cv2.resize(a, (2, 28), interpolation=cv2.INTER_NEAREST)
        np.testing.assert_array_equal(got, a[LO.nearest_dsize(n, 28)], err_msg="n=%d -> 28" % n)
        pairs += 1
    assert pairs >= 64


def test_roi_boxes_round_half_to_even():
    b = LO.roi_boxes(dict(boxes=np.array([[2.5, 3.5, 2.5, 4.4]], np.float32)), [0], 1.0)
    assert b.tolist() == [[2, 4, 3, 5]]                 # half to even, then the degenerate-side +1


def emulate(L, case):
    """PanopticLabels' host tables applied as the kernel applies them, with the oracle's row spans for mask_gt."""
    import torch
    from upsnet_b200.training import pack_polygons
    e = case["entry"]
    draw, roi_rows = L._rows(e)
    _, _, polys = pack_polygons(e["segms"], draw, "test")

    class P:
        roi_boxes = None
    pk = P()
    if L.with_roi:
        pk.roi_boxes = LO.roi_boxes(e, roi_rows, case["scale"])
    t, n = L.tables(case["label_map"].shape, pk, case["im_shape"], case["scale"], e["flipped"])
    lab = case["label_map"].astype(np.int64)

    def gather(r, c):
        out = lab[np.maximum(r, 0)][:, np.maximum(c, 0)]
        out[r < 0, :] = 255
        out[:, c < 0] = 255
        return out
    out = {"seg_gt": gather(t["seg_rows"], t["seg_cols"])[None],
           "seg_gt_4x": gather(t["q_rows"], t["q_cols"])[None]}
    m = np.zeros((len(polys), len(t["m_rows"]), len(t["m_cols"])), np.int64)
    for g, ps in enumerate(polys):
        edges = [LO.polygon_edges(p) for p in ps]
        for y, Y in enumerate(t["m_rows"]):
            if Y < 0:
                m[g, y] = 255
                continue
            spans = [s for es in edges if es for s in LO.row_spans(es, Y)]
            for x, X in enumerate(t["m_cols"]):
                m[g, y, x] = 255 if X < 0 else int(any(a <= X <= b for a, b in spans))
    out["mask_gt"] = m
    if L.with_roi:
        out["seg_roi_gt"] = np.stack([gather(t["roi_rows"][i * L.M:(i + 1) * L.M], t["roi_cols"][i * L.M:(i + 1) * L.M])
                                      for i in range(n)]) if n else np.zeros((0, L.M, L.M), np.int64)
    return out


@pytest.mark.parametrize("case", [c for c in CASES if c["name"] in ("cs_scale125_flip", "cs_special", "coco_1333_640",
                                                                     "cs_cvround_int", "cs_canvas_mismatch")],
                         ids=lambda c: c["name"])
def test_package_tables_match_reference(case):
    from upsnet_b200 import PanopticLabels, _lib
    L = PanopticLabels(dataset=case["dataset"], with_roi=case["with_roi"])
    if case["raises"]:
        with pytest.raises(_lib.UpsnetError):
            emulate(L, case)
        return
    out = emulate(L, case)
    assert sorted(out) == sorted(case["ref"])
    for k, v in case["ref"].items():
        np.testing.assert_array_equal(out[k], v, err_msg=k)
