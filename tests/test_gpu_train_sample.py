"""TrainingSample on the device against what the reference's loader and collate made of the same roidb entries
(tests/golden/reference_train_sample.npz), the flip of upsnet_prep_image against a host-flipped copy, and one reduced
training step fed by a flipped, rescaled sample against the float64 oracle of tests/train_forward_oracle.py."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import label_oracle as LO  # noqa: E402
import train_forward_oracle as TF  # noqa: E402
import train_sample_cases as TS  # noqa: E402
from test_gpu_train_forward import _compare, _oracle, _product_step  # noqa: E402
from test_train_sample_cpu import CASES, IDS, sampler  # noqa: E402

pytestmark = pytest.mark.gpu
RPN_PREFIXES = ("rpn_labels_fpn", "rpn_bbox_targets_fpn", "rpn_bbox_inside_weights_fpn", "rpn_bbox_outside_weights_fpn")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda", 0)


@pytest.fixture
def precision():
    from upsnet_b200 import operators as ops
    saved = ops._PRECISION["conv"]
    yield
    ops._PRECISION["conv"] = saved


def bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("h,w,scale", [(37, 53, 1.0), (37, 53, 0.6), (37, 53, 1.7), (61, 99, 0.35), (1, 7, 3.0),
                                       (45, 1, 2.0)])
def test_flipped_prep_is_prep_of_a_flipped_copy(dev, h, w, scale):
    """flip=True equals prep_image of the host-flipped image bit for bit, at scale 1, down and up, odd widths, padding."""
    from upsnet_b200 import prep_image
    im = torch.from_numpy(TS.image_bgr(h, w, h * 131 + w)).to(dev)
    got, hw = prep_image(im, TS.PIXEL_MEANS, scale, flip=True)
    want, hw2 = prep_image(im.flip(1).contiguous(), TS.PIXEL_MEANS, scale)
    assert hw == hw2 and got.shape == want.shape
    assert torch.equal(bits(got), bits(want))
    if w > 1:                                       # and the flag does flip
        same, _ = prep_image(im, TS.PIXEL_MEANS, scale)
        assert not torch.equal(bits(same), bits(got))


def _sample(case, dev, seed):
    h, w = case["shape"]
    image, label_map = TS.image_bgr(h, w, case["image_seed"]), LO.label_png(h, w, case["label_seed"])
    np.random.seed(case["np_seed"])
    return sampler(case["dataset"]).sample(case["entry"], image, label_map, dev, seed=seed)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_sample_vs_reference(dev, case):
    data, label = _sample(case, dev, seed=5)
    # the keys, kinds, dtypes and shapes of collate (data_4x is not built; the RPN fields are checked below)
    want_data = [r for r in case["data_layout"] if not r.startswith("data_4x|")]
    assert [TS.layout_row(k, v) for k, v in sorted(data.items())] == want_data
    rest = {k: v for k, v in label.items() if not k.startswith(RPN_PREFIXES)}
    assert [TS.layout_row(k, v) for k, v in sorted(rest.items())] == case["label_layout"]
    assert data["data"].is_cuda and all(v.is_cuda for v in label.values() if torch.is_tensor(v))
    # im_info, gt_classes and the label maps bit-exact
    assert data["im_info"].tobytes() == case["im_info"].tobytes()
    assert np.array_equal(label["gt_classes"].cpu().numpy(), case["gt_classes"])
    assert sorted(case["digests"]) == sorted(k for k in ("seg_gt", "seg_gt_4x", "mask_gt", "seg_roi_gt") if k in label)
    for k, d in case["digests"].items():
        assert LO.digest({k: label[k].cpu().numpy()}) == d, k
    # the image blob on the fixture's grid: exact without a resize, else within cv2's SIMD rounding
    blob = data["data"][0].cpu().numpy()[:, case["blob_rows"]][:, :, case["blob_cols"]]
    want = case["blob"]
    if float(case["im_scale"]) == 1.0:
        assert np.array_equal(blob.view(np.uint32), want.view(np.uint32))
    else:
        assert np.abs(blob - want).max() < 1e-3 * max(1.0, np.abs(want).max() / 30)


@pytest.mark.parametrize("case", [CASES[1], CASES[6]], ids=[IDS[1], IDS[6]])
def test_rpn_fields_are_rpn_targets(dev, case):
    """The RPN fields equal RPNTargets.from_roidb at the sample's scale and seed; without a seed, it is the np.random
    draw that follows the scale draw (add_rpn_blobs runs after get_image_blob)."""
    from upsnet_b200.training import RPNTargets
    cfg = TS.CONFIGS[case["dataset"]]
    s = float(case["im_scale"])
    for seed in (5, None):
        _, label = _sample(case, dev, seed=seed)
        if seed is None:
            np.random.seed(case["np_seed"])
            np.random.randint(0, high=len(cfg["scales"]), size=1)
            seed = int(np.random.randint(np.iinfo(np.int64).max, dtype=np.int64))
        want = RPNTargets(max_size=cfg["max_size"]).from_roidb(case["entry"], s, dev, seed=seed)
        got = {k: v for k, v in label.items() if k.startswith(RPN_PREFIXES)}
        assert sorted(got) == sorted(want) and len(got) == 20
        for k, v in want.items():
            assert got[k].dtype == v.dtype and got[k].shape == v.shape
            assert torch.equal(got[k].contiguous().view(torch.uint8), v.contiguous().view(torch.uint8)), k


def test_training_step_from_a_flipped_rescaled_sample(dev, precision):
    """One reduced step (R50 widths, depth 2 per stage, bf16x3) on a flipped entry drawn at scale 1.25, against the
    float64 oracle with test_gpu_train_forward's criterion."""
    import upsnet_b200 as U
    from upsnet_b200.synthetic import synthetic_model
    depth = (2, 2, 2, 2)
    m = synthetic_model(depth=depth, seed=1, device=dev)
    base, label_map = TF.synthetic_entry(2, 128, 256, 4)
    entry = TS.flip_entry(base)
    ts = U.TrainingSample(dataset="cityscapes", scales=(160,), max_size=512)
    np.random.seed(0)
    data, label = ts.sample(entry, TS.image_bgr(128, 256, 3), label_map, dev)
    assert float(data["im_info"][0, 2]) == 1.25 and tuple(data["data"].shape) == (1, 3, 160, 320)
    U.set_precision("bf16x3")
    out = _product_step(m, data, label, seed=5)
    want, wgrads = _oracle(m, depth, 100, dev).step(data["data"], label, out["_intermediates"])
    _compare(m, out, want, wgrads, "bf16x3", "sample")


def test_bad_input_raises_before_any_launch(dev):
    from kernel_trace import launched_kernels
    from upsnet_b200._lib import UpsnetError
    case = CASES[6]
    h, w = case["shape"]
    image, label_map = TS.image_bgr(h, w, 1), LO.label_png(h, w, 1)
    ts = sampler(case["dataset"])
    entry = case["entry"]
    no_boxes = dict(entry, boxes=np.zeros((0, 4), np.float32), gt_classes=np.zeros(0, np.int32),
                    is_crowd=np.zeros(0, np.int32), segms=[])
    all_crowd = dict(entry, is_crowd=np.ones_like(entry["is_crowd"]))
    bad = [(entry, image, label_map[:, :-1]), (entry, image[:-1], label_map), (entry, image, label_map.astype(np.int32)),
           (no_boxes, image, label_map), (all_crowd, image, label_map)]

    def run():
        for e, im, lab in bad:
            with pytest.raises(UpsnetError):
                ts.sample(e, im, lab, dev, seed=1)

    def ours(name):                     # the library's kernels (namespace ups) and any copy to or from the device
        return "ups::" in name or "Memcpy" in name

    _, kernels = launched_kernels(run, keep=ours)
    assert not kernels, kernels
    _, control = launched_kernels(lambda: ts.sample(entry, image, label_map, dev, seed=1), keep=ours)
    assert any("prep_image" in k for k in control) and any("Memcpy" in k for k in control), control
