"""The training-forward oracle (tests/train_forward_oracle.py) on a tiny model on the CPU: its float64 gradients reject
planted faults under the criterion the GPU test applies, and get_params_lr() follows the reference's grouping rule."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import train_forward_oracle as TF  # noqa: E402


def _decisions(entry, H, W, seed, K=9, S=19, R=48, M=28):
    """Discrete decisions and loader labels of one step, drawn at random (the GPU tests take them from the product)."""
    rng = np.random.default_rng(seed)
    f32 = np.float32
    xy = np.sort(rng.uniform(0, [W - 1, H - 1, W - 1, H - 1], (R, 4)).reshape(R, 2, 2), axis=1).reshape(R, 4)
    xy = xy[:, [0, 1, 2, 3]]
    boxes = np.stack([np.minimum(xy[:, 0], xy[:, 2]), np.minimum(xy[:, 1], xy[:, 3]),
                      np.maximum(xy[:, 0], xy[:, 2]) + 4, np.maximum(xy[:, 1], xy[:, 3]) + 4], 1).clip(0, W - 1)
    rois = torch.from_numpy(np.hstack([np.zeros((R, 1)), boxes]).astype(f32))
    labels = rng.integers(0, K, R)
    labels[R // 2:] = 0
    tgt = np.zeros((R, 4 * K), f32)
    iw = np.zeros((R, 4 * K), f32)
    for i, c in enumerate(labels):
        if c > 0:
            tgt[i, 4 * c:4 * c + 4] = rng.standard_normal(4)
            iw[i, 4 * c:4 * c + 4] = 1
    nm = int((labels > 0).sum())
    mt = rng.integers(-1, 2, (nm, K * M * M)).astype(f32)
    t = {"rois": rois, "labels": torch.from_numpy(labels), "bbox_targets": torch.from_numpy(tgt),
         "bbox_inside_weights": torch.from_numpy(iw), "bbox_outside_weights": torch.from_numpy((iw > 0).astype(f32)),
         "mask_rois": rois[:R // 2][torch.from_numpy(labels[:R // 2] > 0)], "mask_int32": torch.from_numpy(mt)}
    G = entry["boxes"].shape[0]
    keep = np.sort(rng.permutation(G)[:max(int(G * 0.7), 1)])
    gt = torch.from_numpy(np.hstack([np.zeros((G, 1), f32), entry["boxes"]]).astype(f32))
    inter = {"proposal_targets": t, "gt_rois": gt[torch.from_numpy(keep)],
             "cls_idx": torch.from_numpy(entry["gt_classes"].astype(np.int64))[torch.from_numpy(keep)], "keep_inds": keep}
    label = {}
    for s in TF.STRIDES:
        Fh, Fw = -(-H // s), -(-W // s)
        label["rpn_labels_fpn%d" % s] = torch.from_numpy(rng.integers(-1, 2, (1, 3, Fh, Fw)))
        label["rpn_bbox_targets_fpn%d" % s] = torch.from_numpy(rng.standard_normal((1, 12, Fh, Fw)).astype(f32))
        w_ = (rng.random((1, 12, Fh, Fw)) < 0.1).astype(f32)
        label["rpn_bbox_inside_weights_fpn%d" % s] = torch.from_numpy(w_)
        label["rpn_bbox_outside_weights_fpn%d" % s] = torch.from_numpy(w_ / 64)
    seg = rng.integers(0, S, (1, H, W))
    seg[rng.random((1, H, W)) < 0.1] = 255
    label["seg_gt"] = torch.from_numpy(seg)
    label["seg_gt_4x"] = torch.from_numpy(seg[:, ::4, ::4].copy())
    label["mask_gt"] = torch.from_numpy((rng.random((G, H // 4, W // 4)) < 0.2).astype(np.uint8))
    inter["fcn_rois"] = gt                      # the ROI loss takes every ground-truth box, before the keep draw
    seg_roi = rng.integers(0, S, (G, M, M))
    seg_roi[rng.random((G, M, M)) < 0.2] = 255
    label["seg_roi_gt"] = torch.from_numpy(seg_roi)
    return inter, label


def _tiny(cfg=None, K=9, S=19):
    from upsnet_b200.synthetic import synthetic_model
    with torch.random.fork_rng(devices=[]):
        m = synthetic_model(cfg, depth=(2, 2, 2, 2), seed=3)
    H, W = 64, 96
    entry, _ = TF.synthetic_entry(5, H, W, 5, num_classes=K)
    inter, label = _decisions(entry, H, W, 7, K, S)
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    return sd, TF.trainable_names(m), TF.image(11, H, W), inter, label


def _run(tiny, dtype=torch.float64, fault=None, **kw):
    sd, names, img, inter, label = tiny
    return TF.TrainOracle(sd, names, dtype=dtype, fault=fault, **kw).step(img, label, inter)


# the oracle of UPSNetConfig.coco_r50's structure: FPN's global context branch and the semantic head's ROI loss
COCO = dict(num_classes=81, num_seg_classes=133, fcn_layers=3, with_gap=True, fcn_with_roi_loss=True)


@pytest.fixture(scope="module")
def tiny():
    return _tiny()


@pytest.fixture(scope="module")
def clean(tiny):
    return _run(tiny)


@pytest.fixture(scope="module")
def coco():
    """(the tiny step of a coco_r50-structured model, its clean oracle step)"""
    from upsnet_b200.model import UPSNetConfig
    tiny = _tiny(UPSNetConfig.coco_r50(), K=81, S=133)
    return tiny, _run(tiny, **COCO)


def test_fp32_oracle_passes_criterion(tiny, clean):
    out, g = _run(tiny, torch.float32)
    err = TF.grad_errors(g, clean[1])
    assert all(e <= TF.grad_tol(k, "bf16x3") for k, e in err.items()), sorted(err.items(), key=lambda kv: -kv[1])[:3]
    for k in TF.LOSSES:
        assert abs(out[k] - clean[0][k]) <= TF.LOSS_TOL["bf16x3"] * max(abs(clean[0][k]), 1e-3), k


@pytest.mark.parametrize("fault", TF.FAULTS + TF.COCO_FAULTS)
def test_planted_fault_rejected(request, fault):
    if fault in TF.COCO_FAULTS:
        (tiny, clean), kw = request.getfixturevalue("coco"), COCO
    else:
        tiny, clean, kw = request.getfixturevalue("tiny"), request.getfixturevalue("clean"), {}
    _, g = _run(tiny, fault=fault, **kw)
    err = TF.grad_errors(g, clean[1])
    assert any(e > TF.grad_tol(k, "bf16x3") for k, e in err.items()), fault


def test_get_params_lr_matches_reference_rule():
    from upsnet_b200.model import resnet_upsnet
    m = resnet_upsnet([2, 2, 2, 2])
    groups = m.get_params_lr()
    assert len(groups) == 13
    assert groups[0]["params"] == [] and groups[0]["lr"] == 1 and groups[0]["weight_decay"] == 0
    name = {id(p): n for n, p in m.named_parameters()}
    mods = [("resnet_backbone.res3", "resnet_backbone.res4", "resnet_backbone.res5"), ("fpn",), ("rcnn",),
            ("mask_branch",), ("rpn",), ("fcn_head",)]
    for i, prefixes in enumerate(mods):
        for j, suffix in enumerate(("weight", "bias")):
            g = groups[1 + 2 * i + j]
            want = [n for n, p in m.named_parameters() if n.startswith(tuple(p_ + "." for p_ in prefixes))
                    and n.split(".")[-1] == suffix and ".bn" not in n and "downsample.1" not in n]
            assert [name[id(p)] for p in g["params"]] == want
            assert g["lr"] == (1 if suffix == "weight" else 2)
            assert ("weight_decay" in g) == (suffix == "bias") and g.get("weight_decay", 0) == 0
    listed = {id(p) for g in groups for p in g["params"]}
    for n, p in m.named_parameters():
        assert (id(p) in listed) == p.requires_grad, n
        frozen = n.startswith(("resnet_backbone.conv1.", "resnet_backbone.res2.")) or ".bn" in n or "downsample.1" in n
        assert p.requires_grad != frozen, n


def test_fcn_with_roi_loss_raises_before_any_launch():
    from upsnet_b200._lib import UpsnetError
    from upsnet_b200.model import UPSNetConfig, resnet_upsnet
    m = resnet_upsnet([2, 2, 2, 2], UPSNetConfig(fcn_with_roi_loss=True))
    data = {"data": torch.zeros(1, 3, 64, 64), "im_info": np.array([[64, 64, 1.0]], np.float32)}
    with pytest.raises(UpsnetError, match="fcn_with_roi_loss"):
        m(data, {"roidb": {}})
    assert UPSNetConfig.coco_r101_dcn().fcn_with_roi_loss


def test_freeze_config_sets_requires_grad_and_training_needs_freeze_at_2():
    from upsnet_b200._lib import UpsnetError
    from upsnet_b200.model import UPSNetConfig, resnet_upsnet

    class Cfg(dict):
        def __getattr__(self, k):
            if k not in self:
                raise AttributeError(k)
            return self[k]
    ref = Cfg(network=Cfg(backbone_freeze_at=3, backbone_fix_bn=True), train=Cfg(), test=Cfg(), dataset=Cfg())
    cfg = UPSNetConfig.from_reference_config(ref)
    assert cfg.backbone_freeze_at == 3 and cfg.backbone_fix_bn
    m = resnet_upsnet([2, 2, 2, 2], cfg)
    for n, p in m.named_parameters():
        frozen = n.startswith(("resnet_backbone.conv1.", "resnet_backbone.res2.", "resnet_backbone.res3.")) or \
            ".bn" in n or "downsample.1" in n
        assert p.requires_grad != frozen, n
    data = {"data": torch.zeros(1, 3, 64, 64), "im_info": np.array([[64, 64, 1.0]], np.float32)}
    with pytest.raises(UpsnetError, match="freeze_at"):
        m(data, {"roidb": {}})
    m = resnet_upsnet([2, 2, 2, 2], UPSNetConfig(backbone_fix_bn=False))
    assert all(p.requires_grad for n, p in m.named_parameters() if ".bn" in n and ".res3." in n)
    with pytest.raises(UpsnetError, match="fix_bn"):
        m(data, {"roidb": {}})


def test_prepare_forgets_the_parameters_in_every_weight_cache():
    """An optimiser step replayed from a CUDA graph leaves the parameters' versions as they were, so the model forgets
    what every per-weight cache, the training dgrad packs included, holds for its parameters; other entries stay."""
    from upsnet_b200 import operators as ops, training
    from upsnet_b200.model import resnet_upsnet
    m = resnet_upsnet([2, 2, 2, 2])
    w, other = m.rpn.cls_score.weight, torch.zeros(2, 3)
    assert training._dgrad_cache in ops._weight_caches
    for cache in ops._weight_caches:
        for t in (w, other):
            ops._per_weight(cache, t, lambda: "packed")
    m.prepare()
    assert all(id(w) not in c and id(other) in c for c in ops._weight_caches)
