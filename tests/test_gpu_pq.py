"""Device PQ statistics (csrc/pq.cu) and label-map restore (upsnet_label_restore) against the reference fixtures
(tests/golden/reference_pq.npz) and the numpy oracle, plus the engine's restore_size path end to end."""
import os

import numpy as np
import pytest
import torch

import pq_oracle as P
from oracle import oracle as O

pytestmark = pytest.mark.gpu

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_pq.npz"))
CATS = {int(c): {'id': int(c), 'isthing': int(t)} for c, t in zip(GOLD["cat_ids"], GOLD["cat_isthing"])}
CASES = [str(c) for c in GOLD["cases"]]
DEV = torch.device("cuda", 0)


def case_images(name):
    out = []
    for k in range(int(GOLD[name + "/n"])):
        segs = [{"id": int(r[0]), "category_id": int(r[1]), "iscrowd": int(r[2]), "area": int(r[3])}
                for r in GOLD["%s/%d/segs" % (name, k)]]
        out.append((GOLD["%s/%d/pan" % (name, k)], GOLD["%s/%d/gt" % (name, k)], segs))
    return out


def device_stat(pq):
    torch.cuda.synchronize()
    a = np.zeros((256, 4))
    a[:, 0] = pq._iou.cpu().numpy()
    a[:, 1:] = pq._counts.cpu().numpy().T
    return a


def oracle_stat(images):
    stat = {}
    for pan, gt, segs in images:
        P.pq_image(pan, gt, segs, CATS, stat)
    a = np.zeros((256, 4))
    for c, v in stat.items():
        a[c] = v
    return a


def check_stat(got, want):
    assert np.array_equal(got[:, 1:], want[:, 1:])
    assert (np.abs(got[:, 0] - want[:, 0]) <= 1e-12 * np.maximum(want[:, 1], 1)).all()


def random_case(rng, H=1024, W=2048, n_gt=400, n_pred=150):
    """Seeded synthetic image: stuff bands plus n_gt thing rectangles (random ids, ~10 % crowd, VOID holes, some ids
    missing from the table, one duplicate entry), and a prediction that copies and shifts about half of them with
    instance numbers up to 255, adds n_pred others, relabels some stuff, and has stray stuff instances and void."""
    gid = np.zeros((H, W), np.int64)
    ids = rng.choice(np.arange(1, 1 << 24), n_gt + 11, replace=False)
    cats, crowd = {}, set()
    band = H // 11 + 1
    cls = np.zeros((H, W), np.int64)
    for k in range(11):
        gid[k * band:(k + 1) * band] = ids[k]
        cats[int(ids[k])] = k
        cls[k * band:(k + 1) * band] = k if rng.random() > 0.15 else (k + 1) % 11
    ins = rng.integers(0, 4, (H, W)) * (rng.random((H, W)) < 0.01)
    for i in ids[11:]:
        h, w = int(rng.integers(4, H // 6)), int(rng.integers(4, W // 6))
        y, x = int(rng.integers(0, H - h)), int(rng.integers(0, W - w))
        gid[y:y + h, x:x + w] = i
        cats[int(i)] = int(rng.integers(11, 19))
        if rng.random() < 0.1:
            crowd.add(int(i))
    for j in range(n_pred):
        h, w = int(rng.integers(4, H // 6)), int(rng.integers(4, W // 6))
        y, x = int(rng.integers(0, H - h)), int(rng.integers(0, W - w))
        cls[y:y + h, x:x + w] = int(rng.integers(11, 19))
        ins[y:y + h, x:x + w] = 1 + j % 255
    for i in ids[11:][: n_gt // 2]:
        ys, xs = np.nonzero(gid == i)
        if ys.size:
            dy, dx = rng.integers(-3, 4, 2)
            cls[np.clip(ys + dy, 0, H - 1), np.clip(xs + dx, 0, W - 1)] = cats[int(i)]
            ins[np.clip(ys + dy, 0, H - 1), np.clip(xs + dx, 0, W - 1)] = int(rng.integers(1, 256))
    cls[rng.random((H, W)) < 0.03] = 255
    gid[rng.random((H, W)) < 0.03] = 0
    present = set(np.unique(gid).tolist()) - {0}
    segs = [{"id": i, "category_id": c, "iscrowd": int(i in crowd), "area": int((gid == i).sum())}
            for i, c in cats.items() if i in present and rng.random() > 0.03]
    segs.append(dict(segs[len(segs) // 2], area=segs[len(segs) // 2]["area"] + 5))
    pan = np.stack([cls, np.minimum(ins, 255), np.zeros_like(cls)], -1).astype(np.uint8)
    gt = np.stack([gid % 256, (gid // 256) % 256, gid // 65536], -1).astype(np.uint8)
    return pan, gt, segs


@pytest.mark.parametrize("name", CASES)
def test_pq_kernel_matches_reference_fixture(name):
    from upsnet_b200 import PanopticQuality
    pq = PanopticQuality(CATS)
    imgs = case_images(name)
    for pan, gt, segs in imgs:
        pq.update(pan, gt, segs)
    check_stat(device_stat(pq), GOLD[name + "/stat"])
    if int(GOLD[name + "/raises"]):
        with pytest.raises(ZeroDivisionError):
            pq.summarize()
        return
    res = pq.summarize()
    for r, key in enumerate(("All", "Things", "Stuff")):
        want = GOLD[name + "/summary"][r]
        assert res[key]["n"] == int(want[3])
        assert np.allclose([res[key]["pq"], res[key]["sq"], res[key]["rq"]], want[:3], rtol=1e-12, atol=1e-14)
    pc = GOLD[name + "/per_class"]
    for c, v in res["per_class"].items():
        assert np.allclose([v["pq"], v["sq"], v["rq"]], pc[c], rtol=1e-12, atol=1e-14)


def test_pq_kernel_random_large_vs_oracle_accumulated_and_bit_identical():
    from upsnet_b200 import PanopticQuality
    rng = np.random.default_rng(7)
    imgs = [random_case(rng) for _ in range(8)]
    for pan, gt, segs in imgs[:2]:                 # one image at a time
        pq = PanopticQuality(CATS)
        pq.update(torch.from_numpy(pan).to(DEV), torch.from_numpy(gt).to(DEV), segs, check_errors=True)
        check_stat(device_stat(pq), oracle_stat([(pan, gt, segs)]))
    runs = []
    for _ in range(2):                             # 8-image accumulation, twice: bit-identical accumulators
        pq = PanopticQuality(CATS)
        for pan, gt, segs in imgs:
            pq.update(pan, gt, segs)
        pq.check_errors()
        runs.append((pq._counts.clone(), pq._iou.clone()))
        check_stat(device_stat(pq), oracle_stat(imgs))
    assert torch.equal(runs[0][0], runs[1][0])
    assert torch.equal(runs[0][1].view(torch.int64), runs[1][1].view(torch.int64))


def test_pq_error_flags_raise():
    from upsnet_b200 import PanopticQuality
    from upsnet_b200._lib import UpsnetError
    pan, gt, segs = case_images("perfect")[0]
    pq = PanopticQuality(CATS)
    bad = pan.copy()
    bad[3, 5, 0] = 200                             # class 200: not a category (the reference raises KeyError)
    with pytest.raises(KeyError):
        pq.update(bad, gt, segs, check_errors=True)
    with pytest.raises(KeyError):
        pq.summarize()                             # sticky
    pq.reset()
    pq.update(pan, gt, segs, check_errors=True)
    many = [{"id": i + 1, "category_id": 3, "iscrowd": 0, "area": 1} for i in range(4097)]
    pq.update(pan, gt, many)
    with pytest.raises(UpsnetError, match="ground-truth segments"):
        pq.check_errors()
    pq.reset()
    pq.update(pan, gt, many[:4096], check_errors=True)    # the limit itself is fine


def test_pq_update_captures_in_cuda_graph():
    from upsnet_b200 import PanopticQuality
    rng = np.random.default_rng(3)
    pan, gt, segs = random_case(rng, 256, 512, 60, 30)
    pan_d, gt_d = torch.from_numpy(pan).to(DEV), torch.from_numpy(gt).to(DEV)
    pq = PanopticQuality(CATS)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(PanopticQuality.STAGING_SLOTS + 1):
            pq.update(pan_d, gt_d, segs)           # warm-up outside the capture; every staging slot has been used
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    pq.reset()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):                      # raises if update() synchronises with the host
        pq.update(pan_d, gt_d, segs)
    torch.cuda.synchronize()
    assert int(pq._counts.abs().sum()) == 0        # captured, not run
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    want = oracle_stat([(pan, gt, segs)] * 3)
    check_stat(device_stat(pq), want)
    pq.update(pan_d, gt_d, segs)                   # the ring still works after a slot went to the graph
    check_stat(device_stat(pq), oracle_stat([(pan, gt, segs)] * 4))


@pytest.mark.parametrize("k", range(int(GOLD["restore/n"])))
def test_label_restore_matches_cv2_fixture(k):
    import upsnet_b200 as U
    Hp, Wp = (int(v) for v in GOLD["restore/%d/shape" % k])
    lab = P.restore_label(Hp, Wp, k)
    info = GOLD["restore/%d/im_info" % k]
    want_sha = str(GOLD["restore/%d/want_sha256" % k])                    # digest of cv2.resize's output
    got = U.label_restore(torch.from_numpy(lab).to(DEV), info)
    assert got.shape == (1,) + tuple(GOLD["restore/%d/want_shape" % k]) and got.dtype == torch.int64
    assert P.digest(got[0].cpu().numpy()) == want_sha
    other = (lab * 7 + 3) % 400 - 10
    a, b = U.label_restore(torch.from_numpy(lab[0]).to(DEV), info, torch.from_numpy(other[0]).to(DEV))
    assert P.digest(a.cpu().numpy()) == want_sha
    assert np.array_equal(b.cpu().numpy(), P.label_restore(other, info))


def test_label_restore_random_vs_oracle():
    import upsnet_b200 as U
    rng = np.random.default_rng(11)
    for Hp, Wp, h, w, scale in ((1344, 1344, 800, 1333, 1.0 / 0.75), (1024, 2048, 1024, 2048, 1.0), (96, 128, 77, 101, 0.8),
                                (64, 64, 31, 45, 2.5), (1312, 2144, 1280, 2133, 1.6)):
        lab = rng.integers(-300, 600, (1, Hp, Wp)).astype(np.int64)
        info = np.array([[h, w, scale]], np.float32)
        got = U.label_restore(torch.from_numpy(lab).to(DEV), info)
        assert np.array_equal(got[0].cpu().numpy(), P.label_restore(lab, info))


def _self_gt(pan_2ch, cats):
    """Ground truth equal to the prediction: one gt segment per prediction segment, id = 1 + its rank."""
    cls = pan_2ch[..., 0].astype(np.int64)
    ins = np.where(np.array([bool(cats.get(c, {'isthing': 0})['isthing']) for c in range(256)])[cls], pan_2ch[..., 1], 0)
    key = np.where(cls == 255, -1, cls * 256 + ins)
    keys, inv, cnt = np.unique(key, return_inverse=True, return_counts=True)
    ids = np.zeros(keys.shape, np.int64)
    segs = []
    for r, (kk, n) in enumerate(zip(keys, cnt)):
        if kk < 0:
            continue
        ids[r] = r + 1
        segs.append({"id": r + 1, "category_id": int(kk // 256), "iscrowd": 0, "area": int(n)})
    gid = ids[inv.reshape(cls.shape)]
    gt = np.stack([gid % 256, (gid // 256) % 256, gid // 65536], -1).astype(np.uint8)
    return gt, segs, sorted({s["category_id"] for s in segs})


def test_engine_restore_size_end_to_end():
    import upsnet_b200 as U
    from upsnet_b200 import operators as ops
    from upsnet_b200.model import UPSNetConfig
    from upsnet_b200.synthetic import synthetic_model
    m = synthetic_model(UPSNetConfig.cityscapes_r50(), depth=(1, 1, 1, 1), seed=3, device=DEV)
    H, W, scale = 200, 300, 1.25                  # network input 250 x 375, padded to 256 x 384
    rng = np.random.default_rng(5)
    means = U.PipelinedEngine.PIXEL_MEANS
    raws = [torch.from_numpy(rng.integers(0, 256, (H, W, 3)).astype(np.uint8)).pin_memory() for _ in range(2)]
    im_info = np.array([[250, 375, scale]], np.float32)
    cats = {c: {'id': c, 'isthing': int(c >= 11)} for c in range(19)}
    U.set_precision("bf16x3")
    try:
        plain = U.PipelinedEngine(m, im_info, depth=2, with_unified=True, stuff_area_limit=256, im_scale=scale)
        rest = U.PipelinedEngine(m, im_info, depth=2, with_unified=True, stuff_area_limit=256, im_scale=scale,
                                 restore_size=True)
        for raw in raws:
            a = {k: v.clone() for k, v in plain.result(plain.submit(raw)).items()}
            b = {k: v.clone() for k, v in rest.result(rest.submit(raw)).items()}
            blob, _ = ops.prep_image(raw.to(DEV), means, scale)
            with torch.no_grad():
                want = m({"data": blob, "im_info": im_info})
            # restore_size=False: today's outputs, at the padded network resolution
            assert a["fcn_outputs"].shape == (1, 256, 384)
            assert torch.equal(a["fcn_outputs"], want["fcn_outputs"].cpu())
            assert torch.equal(a["panoptic_outputs"], want["panoptic_outputs"].cpu())
            cls = want["panoptic_cls_inds"].cpu().numpy()
            uni = O.unified_pan_result(want["fcn_outputs"][0].cpu().numpy(), want["panoptic_outputs"][0].cpu().numpy(), cls, 19, 9, 256)
            assert np.array_equal(a["pan_2ch"].numpy(), uni)
            # restore_size=True: label maps and pan_2ch at the original size, pan_2ch computed from the restored maps
            seg_r = P.label_restore(want["fcn_outputs"].cpu().numpy(), im_info)
            pan_r = P.label_restore(want["panoptic_outputs"].cpu().numpy(), im_info)
            assert b["fcn_outputs"].shape == (1, H, W) and b["pan_2ch"].shape == (H, W, 3)
            assert np.array_equal(b["fcn_outputs"][0].numpy(), seg_r)
            assert np.array_equal(b["panoptic_outputs"][0].numpy(), pan_r)
            assert np.array_equal(b["pan_2ch"].numpy(), O.unified_pan_result(seg_r, pan_r, cls, 19, 9, 256))
            # PQ of the prediction against itself as ground truth: exactly 1 for every present category
            gt, segs, present = _self_gt(b["pan_2ch"].numpy(), cats)
            pq = U.PanopticQuality(cats)
            pq.update(b["pan_2ch"], gt, segs, check_errors=True)
            res = pq.summarize()
            assert present
            for c in present:
                v = res["per_class"][c]
                assert v["pq"] == 1.0 and v["sq"] == 1.0 and v["rq"] == 1.0 and v["fp"] == 0 and v["fn"] == 0
    finally:
        U.set_precision("fp32")
