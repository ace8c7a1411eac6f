"""Device confusion matrix (csrc/sseg.cu, SegmentationIoU) against the reference fixtures (tests/golden/reference_sseg.npz)
and the numpy oracle: exact matrices for uint8 and int64 predictions and both class counts, the im_info path against
label_restore + update, full-size images, accumulation, reset, CUDA-graph capture, repeatability and rejected inputs."""
import os

import numpy as np
import pytest
import torch

import sseg_oracle as S

pytestmark = pytest.mark.gpu

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_sseg.npz"))
CASES = [str(c) for c in GOLD["cases"]]
DEV = torch.device("cuda", 0)


def case_images(name):
    out = []
    for k in range(int(GOLD[name + "/n"])):
        key = "%s/%d/im_info" % (name, k)
        out.append((GOLD["%s/%d/pred" % (name, k)], GOLD["%s/%d/gt" % (name, k)], GOLD[key] if key in GOLD.files else None))
    return out


def oracle_matrix(images, C):
    m = np.zeros((C, C))
    for pred, gt, info in images:
        m += S.confusion(pred, gt, C, info)
    return m


@pytest.mark.parametrize("pred_dtype", ["as_stored", "uint8"])
@pytest.mark.parametrize("name", CASES)
def test_sseg_kernel_matches_reference_fixture(name, pred_dtype):
    from upsnet_b200 import SegmentationIoU
    C = int(GOLD[name + "/C"])
    imgs = case_images(name)
    if pred_dtype == "uint8":                      # np.uint8 first: the same matrix, since the kernel wraps int64 alike
        imgs = [(p.astype(np.uint8), g, i) for p, g, i in imgs]
    miou = SegmentationIoU(C)
    for pred, gt, info in imgs:
        miou.update(pred, gt, im_info=info)
    res = miou.summarize()
    want = GOLD[name + "/matrix"]
    assert np.array_equal(res["confusion_matrix"], want)
    assert np.array_equal(res["confusion_matrix"], oracle_matrix(imgs, C))
    assert S.log_lines(res) == [str(s) for s in GOLD[name + "/lines"]]
    ref = S.summarize(want)
    assert np.array_equal(res["IU_array"], ref["IU_array"]) and res["meanIU"] == ref["meanIU"]


@pytest.mark.parametrize("name", ["netres", "netres_coco"])
def test_sseg_im_info_path_equals_label_restore_then_update(name):
    import upsnet_b200 as U
    C = int(GOLD[name + "/C"])
    pred, gt, info = case_images(name)[0]
    a, b = U.SegmentationIoU(C), U.SegmentationIoU(C)
    d = torch.from_numpy(pred).to(DEV)
    a.update(d, gt, im_info=info)
    b.update(U.label_restore(d, info), gt)
    assert torch.equal(a._acc, b._acc)
    assert np.array_equal(a.confusion_matrix(), GOLD[name + "/matrix"])
    rng = np.random.default_rng(4)                 # COCO geometry at full size, restored size one pixel off the gt
    lab = torch.from_numpy(rng.integers(-50, 400, (1, 1344, 1344))).to(DEV)
    info = np.array([800, 1199, 800 / 427], np.float32)
    gt = rng.integers(0, 256, (426, 641)).astype(np.uint8)
    a.reset(), b.reset()
    a.update(lab, gt, im_info=info)
    b.update(U.label_restore(lab, info), gt)
    assert torch.equal(a._acc, b._acc)
    assert np.array_equal(a.confusion_matrix(), S.confusion(lab.cpu().numpy(), gt, C, info))


def test_sseg_large_rebuilt_case_and_coco_size_vs_oracle_bit_identical():
    from upsnet_b200 import SegmentationIoU
    pred, gt = S.synthetic_case(0, 1024, 2048, 19)
    runs = []
    for dtype in (np.int64, np.int64, np.uint8):
        miou = SegmentationIoU(19)
        miou.update(torch.from_numpy(pred.astype(dtype)).to(DEV), torch.from_numpy(gt).to(DEV))
        runs.append(miou.confusion_matrix())
    assert np.array_equal(runs[0], GOLD["large/matrix"])
    assert np.array_equal(runs[0], runs[1]) and np.array_equal(runs[0], runs[2])
    for k, (H, W, ph, pw) in enumerate(((800, 1333, 800, 1333), (640, 1066, 800, 1333), (427, 640, 800, 1199))):
        pred, gt = S.synthetic_case(k + 1, H, W, 133, (ph, pw))
        miou = SegmentationIoU(133)
        miou.update(pred[None, None], gt)
        assert np.array_equal(miou.confusion_matrix(), S.confusion(pred, gt, 133)), (H, W, ph, pw)


def test_sseg_accumulation_and_reset():
    from upsnet_b200 import SegmentationIoU
    imgs = [S.synthetic_case(k, 256 + 13 * k, 512 - 7 * k, 19, (250 + 5 * k, 509 - 3 * k)) for k in range(6)]
    miou = SegmentationIoU(19)
    for pred, gt in imgs:
        miou.update(torch.from_numpy(pred).to(DEV), gt)
    want = sum(S.confusion(p, g, 19) for p, g in imgs)
    assert np.array_equal(miou.confusion_matrix(), want)
    miou.reset()
    assert not miou.confusion_matrix().any()
    miou.update(*imgs[2])
    assert np.array_equal(miou.confusion_matrix(), S.confusion(*imgs[2], 19))


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")      # the capture the refused update() leaves empty
def test_sseg_update_captures_in_cuda_graph():
    from upsnet_b200 import SegmentationIoU
    from upsnet_b200._lib import UpsnetError
    pred, gt = S.synthetic_case(3, 512, 1024, 19, (384, 768))
    p, g = torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV)
    p2 = torch.from_numpy(pred[:300, :700].copy()).to(DEV)
    miou = SegmentationIoU(19)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        miou.update(p, g)                          # caches this geometry's index tables outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    miou.reset()
    g1 = torch.cuda.CUDAGraph()
    with pytest.raises(UpsnetError, match="outside the capture"):
        with torch.cuda.graph(g1):
            miou.update(p2, g)                     # an uncached geometry cannot be uploaded inside a capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):                  # raises if update() synchronises with the host
        miou.update(p, g)
    torch.cuda.synchronize()
    assert not miou.confusion_matrix().any()       # captured, not run
    for _ in range(SegmentationIoU.TABLE_CACHE + 2):
        miou.update(p[:, : 700 - _], g)            # evicts the captured geometry from the cache
    miou.reset()
    for _ in range(3):
        graph.replay()
    assert np.array_equal(miou.confusion_matrix(), 3 * S.confusion(pred, gt, 19))


def test_sseg_rejects_bad_inputs():
    from upsnet_b200 import SegmentationIoU
    miou = SegmentationIoU(19)
    gt = np.zeros((8, 8), np.uint8)
    for bad_pred in (np.zeros((8, 8), np.int32), np.zeros((8, 8), np.float32), np.zeros((2, 8, 8), np.int64),
                     np.zeros((8,), np.int64), np.zeros((1, 1, 1, 8, 8), np.int64), np.zeros((0, 8), np.int64)):
        with pytest.raises(ValueError):
            miou.update(bad_pred, gt)
    for bad_gt in (np.zeros((8, 8), np.int64), np.zeros((1, 8, 8), np.uint8), np.zeros((8, 0), np.uint8)):
        with pytest.raises(ValueError):
            miou.update(np.zeros((8, 8), np.int64), bad_gt)
    with pytest.raises(ValueError, match="outside"):
        miou.update(np.zeros((8, 8), np.int64), gt, im_info=np.array([9, 8, 1.0], np.float32))
    for c in (0, 225):
        with pytest.raises(ValueError):
            SegmentationIoU(c)
    assert not miou.confusion_matrix().any()
    SegmentationIoU(224).update(np.full((4, 4), 223, np.int64), np.full((4, 4), 223, np.uint8))    # the limit itself is fine
