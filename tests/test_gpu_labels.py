"""GPU checks of upsnet_b200.PanopticLabels (csrc/labels.cu): bit-exact to what the reference's loaders and collate
computed (tests/golden/reference_labels.npz) and to the numpy oracle (tests/label_oracle.py), the seeded full-size
digests, determinism under repeats and CUDA-graph replay, the limits, the drop-in's dict, and PanopticLoss fed the
device-built labels."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import label_oracle as LO  # noqa: E402
from test_labels_cpu import CASES, GOLD  # noqa: E402

pytestmark = pytest.mark.gpu


def U():
    import upsnet_b200
    return upsnet_b200


def run(L, case, mask_dtype=torch.int64):
    e = case["entry"]
    packed = L.pack_roidb(e, case["scale"], "cuda")
    lab = torch.from_numpy(case["label_map"]).cuda()
    return L(lab, packed, case["im_shape"], case["scale"], e["flipped"], mask_dtype=mask_dtype)


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
@pytest.mark.parametrize("mask_dtype", [torch.uint8, torch.int64], ids=["u8", "i64"])
def test_matches_reference(case, mask_dtype):
    L = U().PanopticLabels(dataset=case["dataset"], with_roi=case["with_roi"])
    if case["raises"]:
        with pytest.raises(U()._lib.UpsnetError):
            run(L, case, mask_dtype)
        return
    out = run(L, case, mask_dtype)
    assert sorted(out) == sorted(case["ref"])
    assert out["mask_gt"].dtype == mask_dtype
    for k, v in case["ref"].items():
        np.testing.assert_array_equal(out[k].cpu().numpy().astype(np.int64), v, err_msg=k)


@pytest.mark.parametrize("dataset", ["cityscapes", "coco"])
@pytest.mark.parametrize("flipped", [False, True])
def test_matches_oracle(dataset, flipped):
    rng = np.random.default_rng(31 + flipped + 2 * (dataset == "coco"))
    for scale in (1.0, 0.5, 800 / 480.0):
        h0, w0 = 72, 96
        e = LO.random_entry(rng, h0, w0, 12, dataset, flipped, max_polys=3, max_verts=40)
        lab = LO.label_png(h0, w0, int(rng.integers(1 << 30)))
        im_shape = (LO.cv_size(h0, scale), LO.cv_size(w0, scale))
        L = U().PanopticLabels(dataset=dataset, with_roi=True)
        try:
            want = LO.labels(e, lab, im_shape, scale, dataset, True)
        except ValueError:          # a box on the border rounds to an empty crop: the reference's cv2.resize raises
            with pytest.raises(U()._lib.UpsnetError):
                L.from_roidb(e, lab, im_shape, scale, "cuda")
            continue
        got = L.from_roidb(e, lab, im_shape, scale, "cuda")
        for k, v in want.items():
            np.testing.assert_array_equal(got[k].cpu().numpy(), v, err_msg="%s scale %r" % (k, scale))


@pytest.mark.parametrize("name", [c[0] for c in LO.FULL])
def test_full_size_digest(name):
    z = np.load(GOLD)
    entry, lab, im_shape, scale, dataset = LO.full_case(name)
    got = U().PanopticLabels(dataset=dataset, with_roi=True).from_roidb(entry, lab, im_shape, scale, "cuda")
    assert LO.digest({k: v.cpu().numpy() for k, v in got.items()}) == str(z["full/" + name])


def test_deterministic_and_graph_replay():
    entry, lab, im_shape, scale, dataset = LO.full_case("coco_g90")
    L = U().PanopticLabels(dataset=dataset, with_roi=True)
    packed = L.pack_roidb(entry, scale, "cuda")
    labd = torch.from_numpy(lab).cuda()
    tab = L.prepare(tuple(labd.shape), packed, im_shape, scale, entry["flipped"], "cuda")
    a = L.launch(labd, packed, tab)
    b = L.launch(labd, packed, tab)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        L.launch(labd, packed, tab)                     # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        c = L.launch(labd, packed, tab)
    for v in c.values():
        v.fill_(7)
    g.replay()
    torch.cuda.synchronize()
    for k in a:
        assert torch.equal(a[k], b[k]) and torch.equal(a[k], c[k]), k


def test_limits_are_errors():
    L = U().PanopticLabels(dataset="cityscapes", with_roi=False)
    ang = np.linspace(0, 2 * np.pi, 1100, endpoint=False)
    big = [float(v) for v in np.stack([30 + 20 * np.cos(ang), 30 + 20 * np.sin(ang)], 1).ravel()]
    e = dict(boxes=np.array([[10, 10, 50, 50]], np.float32), gt_classes=np.array([1]), is_crowd=np.array([0]),
             segms=[[big]], flipped=False)
    with pytest.raises(U()._lib.UpsnetError):
        L.from_roidb(e, np.zeros((64, 64), np.uint8), (64, 64), 1.0, "cuda")
    e["segms"] = [[[1.0, 2.0, 3.0, 4.0]]]                                   # fewer than 6 coordinates
    with pytest.raises(U()._lib.UpsnetError):
        L.from_roidb(e, np.zeros((64, 64), np.uint8), (64, 64), 1.0, "cuda")
    e["segms"] = [{"size": [64, 64], "counts": "x"}]                        # RLE
    with pytest.raises(U()._lib.UpsnetError):
        L.from_roidb(e, np.zeros((64, 64), np.uint8), (64, 64), 1.0, "cuda")
    torch.cuda.synchronize()


def test_from_roidb_dict_matches_collate():
    case = next(c for c in CASES if c["name"] == "coco_800_480")
    got = U().PanopticLabels(dataset="coco", with_roi=True).from_roidb(
        case["entry"], case["label_map"], case["im_shape"], case["scale"], "cuda")
    assert sorted(got) == ["mask_gt", "seg_gt", "seg_gt_4x", "seg_roi_gt"]
    for k, v in got.items():
        assert v.is_cuda and v.dtype == torch.int64 and tuple(v.shape) == case["ref"][k].shape, k
    no_roi = U().PanopticLabels(dataset="coco", with_roi=False).from_roidb(
        case["entry"], case["label_map"], case["im_shape"], case["scale"], "cuda")
    assert sorted(no_roi) == ["mask_gt", "seg_gt", "seg_gt_4x"]


def test_panoptic_loss_with_device_labels():
    from upsnet_b200.training import gt_rois
    rng = np.random.default_rng(77)
    h0, w0, scale = 96, 128, 1.0
    e = LO.random_entry(rng, h0, w0, 6, "cityscapes", False)
    lab = LO.label_png(h0, w0, 77)
    want = LO.labels(e, lab, (h0, w0), scale, "cityscapes")
    got = U().PanopticLabels(dataset="cityscapes", with_roi=False).from_roidb(e, lab, (h0, w0), scale, "cuda")
    rois, cls = gt_rois(e, scale, "cuda")
    h, w = want["seg_gt_4x"].shape[1:]
    g = torch.Generator().manual_seed(3)
    fcn = torch.randn((1, 19, h, w), generator=g).cuda()
    msk = torch.randn((rois.shape[0], 9, 28, 28), generator=g).cuda()
    res = []
    for seg, mgt in ((torch.from_numpy(want["seg_gt_4x"]).cuda(), torch.from_numpy(want["mask_gt"]).cuda()),
                     (got["seg_gt_4x"], got["mask_gt"])):
        f, m = fcn.clone().requires_grad_(True), msk.clone().requires_grad_(True)
        loss, acc = U().PanopticLoss(num_seg_classes=19, num_classes=9, enable_void=False)(f, m, rois, cls, seg, mgt)
        loss.backward()
        res.append([loss.detach(), acc, f.grad, m.grad])
    for a, b in zip(*res):
        assert torch.equal(a, b)
