"""Proposal targets on the device (csrc/proposal_target.cu through upsnet_b200.training.ProposalTargets) against the
reference fixtures (tests/golden/reference_proposal_targets.npz) and the numpy restatement
(tests/proposal_target_oracle.py)."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import proposal_target_oracle as PO  # noqa: E402
from test_proposal_targets_cpu import CASES, Z, case, check_outputs, fixture  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def targets_for(cfg):
    from upsnet_b200.training import ProposalTargets
    return ProposalTargets(num_classes=cfg.num_classes, batch_rois=cfg.batch_rois, fg_fraction=cfg.fg_fraction,
                           fg_thresh=cfg.fg_thresh, bg_thresh_hi=cfg.bg_hi, bg_thresh_lo=cfg.bg_lo,
                           bbox_reg_weights=cfg.weights, mask_size=cfg.M)


def run(rois, e, scale, cfg, seed):
    t = targets_for(cfg)
    out = t.from_roidb(torch.from_numpy(np.ascontiguousarray(rois)).to(DEV), e,
                       np.array([[0, 0, scale]], np.float32), seed=seed)
    return t, {k: v.cpu().numpy() for k, v in zip(PO.NAMES, out)}


@pytest.mark.parametrize("name", CASES)
def test_fixture(name):
    rois, e, scale, cfg, seed = case(name)
    t, got = run(rois, e, scale, cfg, seed)
    check_outputs(got, fixture(name), name)
    want = PO.proposal_targets(rois, e, scale, cfg, seed)
    assert np.array_equal(t.counts.cpu().numpy(), want["counts"])


@pytest.mark.parametrize("name", [c[0] for c in PO.FULL])
def test_full_size_against_oracle(name):
    e, rois, scale, cfg = PO.full_case(name, 0)
    seeds = (int(Z["full/seed"]), 1, 2 ** 62 + 12345) if name == "coco_g15" else (int(Z["full/seed"]),)
    for seed in seeds:
        t, got = run(rois, e, scale, cfg, seed)
        want = PO.proposal_targets(rois, e, scale, cfg, seed)
        check_outputs(got, want, name)
        assert np.array_equal(t.counts.cpu().numpy(), want["counts"])
        if seed == int(Z["full/seed"]):
            assert PO.digest(got) == str(Z["full/%s/sha256" % name])


def test_same_seed_same_bytes_and_graph_replay():
    e, rois, scale, cfg = PO.full_case("coco_g15", 3)
    t = targets_for(cfg)
    r = torch.from_numpy(rois).to(DEV)
    pk = t.pack_roidb(e, DEV)
    a = {k: v.clone() for k, v in t(r, pk, scale, seed=77).items()}
    b = t(r, pk, scale, seed=77)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        t(r, pk, scale, seed=77)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c = t(r, pk, scale, seed=77)
    for v in c.values():
        v.fill_(7)
    graph.replay()
    torch.cuda.synchronize()
    for k in a:
        assert torch.equal(a[k], c[k]), k


def test_errors():
    from upsnet_b200._lib import UpsnetError
    rois, e, scale, cfg, seed = case("typical")
    t = targets_for(cfg)
    crowd_only = dict(e, is_crowd=np.ones_like(e["is_crowd"]))
    with pytest.raises(UpsnetError):
        t.pack_roidb(crowd_only, DEV)
    segm = list(e["segms"])
    i = int(np.flatnonzero(~np.asarray(e["is_crowd"], bool))[0])
    segm[i] = {"size": [10, 10], "counts": "abc"}
    with pytest.raises(UpsnetError):
        t.pack_roidb(dict(e, segms=segm), DEV)
    # no fg and no bg: every proposal in a band that is neither (bg_lo above every overlap below fg_thresh)
    tt = targets_for(PO.config(num_classes=cfg.num_classes, batch_rois=8, fg_fraction=0.5, bg_lo=0.45, fg_thresh=1.5))
    far = np.array([[0, 1000, 1000, 1010, 1010]], np.float32)
    e1 = PO.entry_from_objects([[0, 0, 10, 10]], [1], [1], [{"size": [1, 1], "counts": "x"}], cfg.num_classes)
    e2 = PO.entry_from_objects([[0, 0, 10, 10], [30, 30, 40, 40]], [1, 2], [1, 0],
                               [{"size": [1, 1], "counts": "x"}, [[30, 30, 40, 30, 40, 40]]], cfg.num_classes)
    with pytest.raises(UpsnetError):
        tt.from_roidb(torch.from_numpy(far).to(DEV), e1, np.array([[0, 0, 1]], np.float32), seed=1)
    with pytest.raises(UpsnetError):
        tt.from_roidb(torch.from_numpy(far).to(DEV), e2, np.array([[0, 0, 1]], np.float32), seed=1)
    assert int(tt.counts[3]) == 1
    from upsnet_b200.training import ProposalTargets
    ag = ProposalTargets(num_classes=9, batch_rois=8, cls_agnostic_bbox_reg=True)
    with pytest.raises(UpsnetError):
        ag(torch.from_numpy(far).to(DEV), ag.pack_roidb(e2, DEV), 1.0, seed=1)


def test_drop_in_dtypes_shapes_and_overlay():
    rois, e, scale, cfg, seed = case("coco_like")
    _, got = run(rois, e, scale, cfg, seed)
    want = fixture("coco_like")
    for k in PO.NAMES:
        assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, k
    from upsnet.operators.modules.proposal_mask_target import ProposalMaskTarget
    m = ProposalMaskTarget(cfg.num_classes, 1, cfg.batch_rois, cfg.fg_fraction, cfg.M, 0.5)
    out = m(torch.from_numpy(rois).to(DEV), e, np.array([[0, 0, scale]], np.float32))     # seed from np.random
    assert [tuple(o.shape[1:]) for o in out] == [want[k].shape[1:] for k in PO.NAMES]
    assert [str(o.dtype) for o in out] == ["torch.float32", "torch.int64"] + ["torch.float32"] * 5 + \
        ["torch.uint8", "torch.int64"]
    assert all(o.is_cuda for o in out)
    assert out[1].shape[0] == want["labels"].shape[0] and out[6].shape[0] == want["mask_int32"].shape[0]
