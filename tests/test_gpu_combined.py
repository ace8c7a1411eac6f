"""Device combined panoptic result (csrc/combined.cu, operators.combined_pan_result) against the reference fixtures
(tests/golden/reference_combined.npz) and the numpy oracle (tests/combined_oracle.py), bit-exact: masks given as host
run lengths and as ops.im_post_rle output, int64 and uint8 semantic maps, a device detection count, ignored classes,
every error flag, the seeded 1024x2048 image, the drop-in on a multi-image list, the engine's 'pan_2ch_combined' and
PanopticQuality on the combined map."""
import os

import numpy as np
import pytest
import torch

import combined_oracle as CO
import pq_oracle as P
from oracle import oracle as O
from upsnet_b200 import operators as ops
from upsnet_b200._lib import UpsnetError

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_combined.npz"))
CASES = [str(c) for c in GOLD["cases"]]


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def case(name):
    runs, off = GOLD[name + "/runs"], GOLD[name + "/run_off"]
    p = GOLD[name + "/params"]
    params = (int(p[0]), int(p[1]), float(p[2]), float(p[3]), int(p[4]))
    return (GOLD[name + "/sem"], GOLD[name + "/scores"], GOLD[name + "/cls"],
            [runs[off[d]:off[d + 1]] for d in range(len(off) - 1)], params)


def device_rle(runs):
    cn, rl = CO.pack_runs(runs)
    return t(cn.view(np.int32)), t(rl)


def run(sem, scores, cls, runs, params, sem_dtype=np.int64, n_dev=None, check_errors=True):
    out = ops.combined_pan_result(t(np.asarray(sem).astype(sem_dtype)), t(np.asarray(scores, np.float32)),
                                  t(np.asarray(cls, np.int64)), device_rle(runs), *params, n_dev=n_dev,
                                  check_errors=check_errors)
    return out.cpu().numpy()


@pytest.mark.parametrize("sem_dtype", [np.int64, np.uint8])
@pytest.mark.parametrize("name", CASES)
def test_fixtures(name, sem_dtype):
    sem, scores, cls, runs, params = case(name)
    got = run(sem, scores, cls, runs, params, sem_dtype)
    assert np.array_equal(got, CO.combined_pan_result(sem, scores, cls, runs, *params))
    if int(GOLD[name + "/order_ok"]):
        assert np.array_equal(got, GOLD[name + "/pan"])


def test_int64_semantic_values_wrap():
    sem, scores, cls, runs, params = case("cityscapes_random")
    wide = sem.astype(np.int64) + 256 * np.random.default_rng(1).integers(-3, 4, sem.shape)
    assert np.array_equal(run(wide, scores, cls, runs, params), GOLD["cityscapes_random/pan"])


def test_device_count_and_ignored_classes():
    """Detections past *n_dev and detections of class 0 / >= num_classes never take part, whatever their score."""
    sem, scores, cls, runs, params = case("cityscapes_random")
    H, W = sem.shape
    full = O.rle_counts(np.ones((H, W), np.uint8))
    junk_cls = np.array([0, params[1], params[1] + 5, -1], np.int64)
    sc = np.concatenate([np.float32([0.999] * 4), scores, np.float32([0.999] * 3)])
    cl = np.concatenate([junk_cls, cls, np.array([1, 2, 3], np.int64)])
    rn = [full] * 4 + list(runs) + [full] * 3
    n_real = 4 + len(runs)
    got = run(sem, sc, cl, rn, params, n_dev=t(np.array([n_real], np.int32)))
    assert np.array_equal(got, GOLD["cityscapes_random/pan"])
    # and without n_dev the trailing full-image detections do take part
    assert np.array_equal(run(sem, sc, cl, rn, params), CO.combined_pan_result(sem, sc, cl, rn, *params))


def blob_probs(rng, n, C):
    yy, xx = np.mgrid[0:28, 0:28].astype(np.float32)
    m = np.zeros((n, C, 28, 28), np.float32)
    for i in range(n):
        for c in range(C):
            cx, cy, r = rng.uniform(8, 20), rng.uniform(8, 20), rng.uniform(5, 16)
            m[i, c] = np.clip(1.0 / (1.0 + np.exp(((xx - cx) ** 2 + (yy - cy) ** 2 - r * r) / 18.0)), 0, 1)
    return m


@pytest.mark.parametrize("H,W,nsc,nc", [(256, 384, 19, 9), (200, 333, 133, 81)])
def test_im_post_rle_masks(H, W, nsc, nc):
    """Masks straight from the device's im_post_rle buffers (engine order, mixed classes, a device count) vs the oracle on
    the host-pasted masks."""
    rng = np.random.default_rng(H)
    n, n_real = 60, 52
    c = np.stack([rng.uniform(0, W, n), rng.uniform(0, H, n)], 1)
    s = rng.uniform(10, 150, (n, 2))
    boxes = np.concatenate([c - s / 2, c + s / 2], 1).astype(np.float32)
    probs = blob_probs(rng, n, 1)
    cls = rng.integers(1, nc, n).astype(np.int64)
    scores = np.round(rng.uniform(0.4, 1.0, n), 2).astype(np.float32)                # ties included
    sem = CO.semantic_map(rng, H, W, nsc, block=8)
    n_dev = t(np.array([n_real], np.int32))
    cn, rl, ovf = ops.im_post_rle(t(boxes), t(probs), t(cls), H, W, n_dev=n_dev)
    assert int(ovf.item()) == 0
    runs = [O.rle_counts(m) for m in O.im_post_masks(boxes[:n_real], probs[:n_real], cls[:n_real], H, W)]
    for sem_dtype in (np.int64, np.uint8):
        for st, ft, lim in ((0.6, 0.7, 4096), (0.45, 0.5, 300)):
            got = ops.combined_pan_result(t(sem.astype(sem_dtype)), t(scores), t(cls), (cn, rl), nsc, nc, st, ft, lim,
                                          n_dev=n_dev).cpu().numpy()
            want = CO.combined_pan_result(sem, scores[:n_real], cls[:n_real], runs, nsc, nc, st, ft, lim)
            assert np.array_equal(got, want)
    assert (want[..., 1] > 0).any()


def test_error_flags():
    sem, scores, cls, runs, params = case("order_across_classes")
    H, W = sem.shape
    cn, rl = CO.pack_runs(runs)
    cap = cn.shape[1]

    def call(cn_, rl_, sc=scores, cl=cls, n_dev=None, sem_=sem):
        return ops.combined_pan_result(t(sem_), t(sc), t(cl), (t(cn_.view(np.int32)), t(rl_)), *params, n_dev=n_dev)

    bad = rl.copy(); bad[0] = cap + 1                                  # im_post_rle overflowed its buffer
    with pytest.raises(UpsnetError, match="RLE counts"):
        call(cn, bad)
    short = cn.copy(); short[1, 0] += 1                                 # runs that do not sum to H * W
    with pytest.raises(ValueError, match="do not cover"):
        call(short, rl)
    n = 2049                                                            # more than 2048 detections
    one = O.rle_counts(np.zeros((H, W), np.uint8))
    cnm, rlm = CO.pack_runs([one] * n)
    with pytest.raises(UpsnetError, match="2048"):
        call(cnm, rlm, np.full(n, 0.9, np.float32), np.ones(n, np.int64))
    # ... but a device count of 2048 is fine
    call(cnm, rlm, np.full(n, 0.9, np.float32), np.ones(n, np.int64), n_dev=t(np.array([2048], np.int32)))
    # the errors are sticky bits of one device word: without check_errors nothing syncs or raises
    ops.combined_pan_result(t(sem), t(scores), t(cls), (t(short.view(np.int32)), t(bad)), *params, check_errors=False)
    # a mask of another size is a ValueError, as the reference's broadcast fails
    with pytest.raises(ValueError):
        call(cn, rl, sem_=sem[:-1])
    with pytest.raises(ValueError):
        ops.combined_pan_result(t(np.zeros((4097, 4097), np.uint8)), t(scores), t(cls), (t(cn.view(np.int32)), t(rl)), *params)


def test_large_image_repeatable():
    sem, scores, cls, runs = CO.large_case()
    p = GOLD["large/params"]
    params = (int(p[0]), int(p[1]), float(p[2]), float(p[3]), int(p[4]))
    a = run(sem, scores, cls, runs, params)
    b = run(sem, scores, cls, runs, params, np.uint8)
    assert np.array_equal(a, b)
    assert CO.digest(a) == str(GOLD["large/sha256"])


def test_dropin_multi_image():
    """get_combined_pan_result on ragged per-image lists (the reference's Pool split raises on them under numpy 2) equals
    the per-image fixtures."""
    names = ["cityscapes_random", "no_detections", "several_instances", "full_height", "defaults"]
    nc = 9
    segs, boxes, masks = [], [[] for _ in range(nc)], [[] for _ in range(nc)]
    for name in names:
        sem, scores, cls, runs, params = case(name)
        assert params[:2] == (19, 9) and params[2:4] == (0.6, 0.7)
        H, W = sem.shape
        segs.append(sem.copy())
        boxes[0].append(np.zeros((0, 5), np.float32))
        masks[0].append([])
        for j in range(1, nc):
            sel = np.flatnonzero(cls == j)
            b = np.zeros((sel.size, 5), np.float32)
            b[:, 4] = scores[sel]
            boxes[j].append(b)
            masks[j].append([{"size": [H, W], "counts": O.rle_to_string(runs[d]).decode()} for d in sel])
    for lim in sorted({int(GOLD[n + "/params"][4]) for n in names}):
        got = ops.get_combined_pan_result(segs, boxes, masks, 19, 9, stuff_area_limit=lim)
        assert len(got) == len(names)
        for k, name in enumerate(names):
            if int(GOLD[name + "/params"][4]) == lim:
                assert np.array_equal(got[k], GOLD[name + "/pan"]), name
            assert np.array_equal(segs[k], GOLD[name + "/sem"])               # not modified


def test_panoptic_quality_on_combined_map():
    import upsnet_b200 as U
    sem, scores, cls, runs, params = case("cityscapes_random")
    pan = run(sem, scores, cls, runs, params)
    H, W = sem.shape
    rng = np.random.default_rng(4)
    gid = (pan[..., 0].astype(np.int64) * 7 + pan[..., 1] + 1) * (rng.random((H, W)) < 0.9)
    gid[:, :W // 4] = 5
    segs = [{"id": int(i), "category_id": int(i - 1) // 7 if i != 5 else 2, "iscrowd": int(i % 5 == 0),
             "area": int((gid == i).sum())} for i in np.unique(gid) if i and (int(i) - 1) // 7 < 19]
    gt = np.stack([gid % 256, gid // 256 % 256, gid // 65536], -1).astype(np.uint8)
    cats = {c: {"isthing": int(c >= 11)} for c in range(19)}
    pq = U.PanopticQuality(cats)
    pq.update(t(pan), t(gt), segs, check_errors=True)
    want = P.pq_image(pan, gt, segs, cats)
    got = pq.pq_stat()
    assert sorted(got) == sorted(want)
    for c, (iou, tp, fp, fn) in want.items():
        assert (got[c]["tp"], got[c]["fp"], got[c]["fn"]) == (tp, fp, fn) and abs(got[c]["iou"] - iou) <= 1e-12 * max(tp, 1)


def test_engine_combined_output():
    import upsnet_b200 as U
    from upsnet_b200.model import UPSNetConfig
    from upsnet_b200.synthetic import synthetic_model
    m = synthetic_model(UPSNetConfig.cityscapes_r50(), depth=(1, 1, 1, 1), seed=3, device=DEV)
    H, W = 256, 384
    im_info = np.array([[H, W, 0.8]], np.float32)
    with pytest.raises(ValueError):
        U.PipelinedEngine(m, im_info, with_combined=True)                          # needs restore_size
    with pytest.raises(ValueError):
        U.PipelinedEngine(m, np.array([[771, 771, 2.042384147644043]], np.float32), restore_size=True, with_combined=True)
    rng = np.random.default_rng(12)
    imgs = [torch.from_numpy(rng.standard_normal((1, 3, H, W)).astype(np.float32) * 40).pin_memory() for _ in range(3)]
    U.set_precision("bf16x3")
    try:
        eng = U.PipelinedEngine(m, im_info, depth=2, with_masks=True, restore_size=True, with_combined=True,
                                combined_score_threshold=0.05, stuff_area_limit=256)
        results = []
        for x in imgs:
            results.append({k: v.clone() for k, v in eng.result(eng.submit(x)).items()})
    finally:
        U.set_precision("fp32")
    instances = 0
    for res in results:
        pan = res["pan_2ch_combined"].numpy()
        assert pan.shape == (320, 480, 3)
        boxes = res["pred_boxes"][:, 1:].numpy() / im_info[0, 2]
        probs, cls = res["mask_probs"].numpy(), res["cls_inds"].numpy()
        runs = [O.rle_counts(mk) for mk in O.im_post_masks(boxes, probs, cls, 320, 480)]
        want = CO.combined_pan_result(res["fcn_outputs"][0].numpy(), res["cls_probs"].numpy(), cls, runs, 19, 9, 0.05,
                                      0.7, 256)
        assert np.array_equal(pan, want)
        instances += int((pan[..., 1] > 0).sum())
    assert instances > 0
