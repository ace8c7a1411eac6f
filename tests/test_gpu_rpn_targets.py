"""RPN training targets on the device (csrc/rpn_target.cu through upsnet_b200.training.RPNTargets) against the reference
fixtures (tests/golden/reference_rpn_targets.npz) and the numpy restatement (tests/rpn_target_oracle.py)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import rpn_target_oracle as RO  # noqa: E402
from test_rpn_targets_cpu import CASES, Z, case, check_against_fixture, ulps  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def targets_for(cfg):
    from upsnet_b200.training import RPNTargets
    return RPNTargets(feat_strides=cfg.strides, anchor_scale=cfg.scale, anchor_ratios=cfg.ratios,
                      rcnn_feat_stride=cfg.rcnn_stride, max_size=cfg.max_size, batch_size=cfg.batch,
                      fg_fraction=cfg.fg_fraction, positive_overlap=cfg.pos, negative_overlap=cfg.neg,
                      straddle_thresh=cfg.straddle)


def flat(d, cfg):
    """The label dict -> concatenated flat numpy arrays in blob order."""
    k = dict(labels="rpn_labels_fpn%d", targets="rpn_bbox_targets_fpn%d", inside="rpn_bbox_inside_weights_fpn%d",
             outside="rpn_bbox_outside_weights_fpn%d")
    return {n: np.concatenate([d[f % s].reshape(-1).cpu().numpy() for s in cfg.strides]) for n, f in k.items()}


def compare(got, want, cfg):
    for k in ("labels", "inside", "outside"):
        assert np.array_equal(got[k], want[k]), k
    xy = RO.xy_mask(cfg)
    assert np.array_equal(got["targets"][xy], want["targets"][xy])
    assert ulps(got["targets"][~xy], want["targets"][~xy]).max() <= 4


@pytest.mark.parametrize("name", CASES)
def test_fixture(name):
    entry, scale, cfg, seed = case(name)
    t = targets_for(cfg)
    d = t.from_roidb(entry, scale, DEV, seed=seed)
    check_against_fixture(name, flat(d, cfg))
    want = RO.from_roidb(entry, scale, cfg, seed)["counts"]
    assert np.array_equal(t.counts.cpu().numpy(), want)


@pytest.mark.parametrize("name", [c[0] for c in RO.FULL])
def test_full_size_against_oracle(name):
    entry, scale, cfg = RO.full_case(name, 0)
    t = targets_for(cfg)
    seeds = (int(Z["full/seed"]), 1, 2 ** 62 + 12345) if name.endswith(("g15", "g50")) else (int(Z["full/seed"]),)
    for seed in seeds:
        got = flat(t.from_roidb(entry, scale, DEV, seed=seed), cfg)
        want = RO.from_roidb(entry, scale, cfg, seed)
        compare(got, want, cfg)
        assert np.array_equal(t.counts.cpu().numpy(), want["counts"])
        if seed == int(Z["full/seed"]):
            assert RO.digest(got, cfg) == str(Z["full/%s/sha256" % name])


def test_same_seed_same_bytes_and_graph_replay():
    entry, scale, cfg = RO.full_case("coco_g15", 3)
    t = targets_for(cfg)
    gt, h, w = RO.gt_from_roidb(entry, scale)
    g = torch.from_numpy(gt).to(DEV)
    a = flat(t(g, h, w, seed=77), cfg)
    b = flat(t(g, h, w, seed=77), cfg)
    for k in a:
        assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        t(g, h, w, seed=77)                                    # warm up on the capture stream
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = t(g, h, w, seed=77)
    graph.replay()
    torch.cuda.synchronize()
    c = flat(out, cfg)
    for k in a:
        assert np.array_equal(a[k].view(np.uint8), c[k].view(np.uint8)), k


def test_no_boxes_raises():
    from upsnet_b200._lib import UpsnetError
    t = targets_for(RO.config(max_size=224))
    with pytest.raises(UpsnetError):
        t(torch.zeros((0, 4), dtype=torch.float32, device=DEV), 100, 100, seed=1)
    e = dict(boxes=np.array([[1, 2, 30, 40]], np.float32), gt_classes=np.array([3]), is_crowd=np.array([1]), height=100,
             width=120)
    with pytest.raises(UpsnetError):
        t.from_roidb(e, 1.0, DEV, seed=1)


def test_too_many_boxes_unsupported():
    from upsnet_b200._lib import lib
    t = targets_for(RO.config(max_size=224))
    cell, ws = t._buffers(DEV)
    N = t.num_anchors
    L = len(t.strides)
    gt = torch.zeros((4097, 4), dtype=torch.float32, device=DEV)
    bufs = [torch.empty(N, dtype=torch.int64, device=DEV)] + [torch.empty(4 * N, device=DEV) for _ in range(3)]
    counts = torch.empty(4, dtype=torch.int32, device=DEV)
    rc = lib().upsnet_rpn_targets(gt.data_ptr(), 4097, cell.data_ptr(), (C.c_int * L)(*t.strides),
                                  (C.c_int * L)(*t.field_sizes), L, t.A, 100.0, 100.0, 0.0, 0.7, 0.3, 256, 128, 1,
                                  *[b.data_ptr() for b in bufs], counts.data_ptr(), ws.data_ptr(), ws.numel(), None)
    assert rc == -2


def test_from_roidb_dict_is_cocos():
    entry, scale, cfg, seed = case("typical")
    d = targets_for(cfg).from_roidb(entry, scale, DEV, seed=seed)
    A = len(cfg.ratios)
    want = {}
    for s, F in zip(cfg.strides, RO.field_sizes(cfg)):
        want["rpn_labels_fpn%d" % s] = ((1, A, F, F), torch.int64)
        for k in ("rpn_bbox_targets_fpn%d", "rpn_bbox_inside_weights_fpn%d", "rpn_bbox_outside_weights_fpn%d"):
            want[k % s] = ((1, 4 * A, F, F), torch.float32)
    assert sorted(d) == sorted(want)
    for k, (shape, dtype) in want.items():
        assert tuple(d[k].shape) == shape and d[k].dtype == dtype and d[k].is_cuda, k


def rpn_loss(d, cfg, H, W, seed):
    """RPNLoss restated in float64: sigmoid cross-entropy over labels != -1 / batch, and the sigma-3 smooth L1 weighted by
    the inside / outside weights, on the same seeded head outputs as the fixture generator (CPU torch generator)."""
    g = torch.Generator().manual_seed(seed)
    A = len(cfg.ratios)
    cls, box = 0.0, 0.0
    for s in cfg.strides:
        h, w = -(-H // s), -(-W // s)
        x = torch.randn((1, A, h, w), generator=g).double().numpy()
        p = (torch.randn((1, 4 * A, h, w), generator=g) * 0.5).double().numpy()
        y = d["rpn_labels_fpn%d" % s][:, :, :h, :w].cpu().numpy()
        t = d["rpn_bbox_targets_fpn%d" % s][:, :, :h, :w].cpu().numpy().astype(np.float64)
        wi = d["rpn_bbox_inside_weights_fpn%d" % s][:, :, :h, :w].cpu().numpy().astype(np.float64)
        wo = d["rpn_bbox_outside_weights_fpn%d" % s][:, :, :h, :w].cpu().numpy().astype(np.float64)
        m = y != -1
        bce = np.maximum(x, 0) - x * y + np.log1p(np.exp(-np.abs(x)))
        cls += bce[m].sum() / cfg.batch
        r = np.abs(wi * (p - t))
        box += (np.where(r < 1 / 9.0, r * r * 4.5, r - 0.5 / 9.0) * wo).sum()
    return cls, box


@pytest.mark.parametrize("name", ["typical", "relabelled", "zero_max_box", "g1500"])
def test_rpn_loss_matches_reference(name):
    entry, scale, cfg, seed = case(name)
    d = targets_for(cfg).from_roidb(entry, scale, DEV, seed=seed)
    H, W = (int(v) for v in Z[name + "/im_info"][:2])
    got = rpn_loss(d, cfg, H, W, seed)
    want = Z[name + "/loss"]
    assert np.allclose(got, want, rtol=1e-6, atol=0), (got, want)
