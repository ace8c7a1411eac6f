"""The fused training losses on the device (csrc/train_loss.cu through upsnet_b200.training.SemanticLoss, RPNLoss and
MaskRCNNLoss) against the reference fixtures (tests/golden/reference_train_losses.npz), the fp64 oracle
(tests/train_loss_oracle.py) and the unfused torch composition with autograd."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import train_loss_oracle as TL  # noqa: E402
from test_train_losses_cpu import Z, mrcnn_fixture, rpn_fixture, sem_fixture  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def within(got, want, rel):
    return np.abs(np.asarray(got) - want).max() <= rel * max(np.abs(want).max(), 1e-30)


def rel_ok(got, want, rel):
    return abs(float(got) - float(want)) <= rel * abs(float(want))


# ---- runners: module forward + backward on device copies of a case ----------------------------
def run_sem(c, grad_out=None, seg_dtype=torch.int64):
    from upsnet_b200 import SemanticLoss
    m = SemanticLoss()
    x = t(c["fcn"]).requires_grad_(True)
    loss = m(x, t(c["seg_gt"]).to(seg_dtype))
    (loss if grad_out is None else loss * grad_out).backward()
    n, bad = m.counts.cpu().tolist()
    return dict(loss=float(loss.detach()), n=n, invalid=bad, d_fcn=x.grad.cpu().numpy(), raw=(loss.detach(), x.grad))


def rpn_device(c):
    return ([t(a).requires_grad_(True) for a in c["scores"]], [t(a).requires_grad_(True) for a in c["preds"]],
            {k: t(v) for k, v in c["label"].items()})


def run_rpn(c, batch=256, go=(1.0, 1.0)):
    from upsnet_b200 import RPNLoss
    xs, ps, lab = rpn_device(c)
    cls_loss, bbox_loss = RPNLoss(rpn_batch_size=batch)(xs, ps, lab)
    (go[0] * cls_loss + go[1] * bbox_loss).backward()
    return dict(cls_loss=float(cls_loss.detach()), bbox_loss=float(bbox_loss.detach()),
                d_scores=[x.grad.cpu().numpy() for x in xs], d_preds=[p.grad.cpu().numpy() for p in ps])


def run_mrcnn(c, go=(1.0, 1.0, 1.0)):
    from upsnet_b200 import MaskRCNNLoss
    inp = [t(c[k]) for k in TL.NAMES]
    for i in range(3):
        inp[i].requires_grad_(True)
    m = MaskRCNNLoss()
    cls_loss, bbox_loss, mask_loss, acc = m(*inp)
    (go[0] * cls_loss + go[1] * bbox_loss + go[2] * mask_loss).backward()
    valid, ignored, matches, mw = m.counts.cpu().tolist()
    return dict(cls_loss=float(cls_loss.detach()), bbox_loss=float(bbox_loss.detach()), mask_loss=float(mask_loss.detach()),
                accuracy=float(acc), valid=valid, ignored=ignored, matches=matches, mask_weight=mw,
                d_cls=inp[0].grad.cpu().numpy(), d_bbox=inp[1].grad.cpu().numpy(), d_mask=inp[2].grad.cpu().numpy())


def check_mrcnn(got, want, rel=1e-5):
    for k in ("cls_loss", "bbox_loss", "mask_loss"):
        assert abs(got[k] - want[k]) <= rel * max(abs(want[k]), 1e-30), k
    for k in ("valid", "ignored", "matches", "mask_weight"):
        assert got[k] == want[k], k
    assert np.float32(got["accuracy"]) == np.float32(want["accuracy"])
    for k in ("d_cls", "d_bbox", "d_mask"):
        assert within(got[k], want[k], rel), k


# ---- fixtures of the reference ----------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(TL.SEM_SMALL))
def test_semantic_matches_the_reference_fixture(name):
    p = "sem/%s/" % name
    got = run_sem(sem_fixture(name))
    assert got["n"] == int(Z[p + "n"]) and got["invalid"] == 0
    assert rel_ok(got["loss"], Z[p + "loss"], 1e-5)
    assert within(got["d_fcn"], Z[p + "d_fcn"], 1e-5)


@pytest.mark.parametrize("name", sorted(TL.RPN_SMALL))
def test_rpn_matches_the_reference_fixture(name):
    p = "rpn/%s/" % name
    got = run_rpn(rpn_fixture(name))
    assert rel_ok(got["cls_loss"], Z[p + "cls_loss"], 1e-5) and rel_ok(got["bbox_loss"], Z[p + "bbox_loss"], 1e-5)
    for s, ds, dp in zip(TL.STRIDES, got["d_scores"], got["d_preds"]):
        assert within(ds, Z[p + "d_score%d" % s], 1e-5) and within(dp, Z[p + "d_pred%d" % s], 1e-5)


@pytest.mark.parametrize("name", sorted(TL.MRCNN_SMALL))
def test_mask_rcnn_matches_the_reference_fixture(name):
    p = "mrcnn/%s/" % name
    c = mrcnn_fixture(name)
    got, want = run_mrcnn(c), TL.mask_rcnn(c)
    for k in ("cls_loss", "bbox_loss", "mask_loss"):
        assert abs(got[k] - float(Z[p + k])) <= 1e-5 * max(abs(float(Z[p + k])), 1e-30), k
    assert np.float32(got["accuracy"]) == Z[p + "accuracy"]
    for k in ("valid", "ignored", "matches", "mask_weight"):
        assert got[k] == want[k], k
    for k in ("d_cls", "d_bbox", "d_mask"):
        assert within(got[k], Z[p + k], 1e-5), k


# ---- semantic loss ----------------------------------------------------------------------------
FULL_SEM = (21, 19, 256, 512, (40, 96), 0.05)      # Cityscapes training size: 1024 x 2048 outputs, 255 padding


def test_semantic_full_size_vs_fp64_oracle():
    c = TL.semantic_case(*FULL_SEM)
    got, want = run_sem(c), TL.semantic(c)
    assert got["n"] == want["n"] and got["invalid"] == 0
    assert rel_ok(got["loss"], want["loss"], 1e-5)
    assert within(got["d_fcn"], want["d_fcn"], 2e-5)


def test_semantic_vs_own_upsampler():
    from upsnet_b200 import operators as ops
    c = TL.semantic_case(*FULL_SEM)
    up = ops.upsample_bilinear(t(c["fcn"]), 4).double().cpu()
    want, n, _ = TL.semantic_from_logits(up, c["seg_gt"])
    got = run_sem(c)
    assert got["n"] == n and rel_ok(got["loss"], float(want), 1e-6)


def test_semantic_peak_memory():
    from upsnet_b200 import SemanticLoss
    c = TL.semantic_case(*FULL_SEM)
    x = t(c["fcn"]).requires_grad_(True)
    seg = t(c["seg_gt"]).long()
    m = SemanticLoss()
    m(x, seg).backward()                 # builds the library and allocator pools outside the measured window
    x.grad = None
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    m(x, seg).backward()
    torch.cuda.synchronize()
    grew = torch.cuda.max_memory_allocated() - base
    assert grew < 32 << 20, grew               # one fcn_output alone is 19 * 1024 * 2048 * 4 B = 159 MB


def test_semantic_all_ignored_and_invalid_labels():
    c = TL.semantic_case(22, 7, 10, 12)
    c["seg_gt"][:] = 255
    got = run_sem(c)
    assert np.isnan(got["loss"]) and got["n"] == 0 and got["invalid"] == 0 and not got["d_fcn"].any()
    c = TL.semantic_case(23, 7, 10, 12, invalid=0.15)
    got, want = run_sem(c), TL.semantic(c)
    assert got["invalid"] == want["invalid"] > 0 and got["n"] == want["n"]
    assert rel_ok(got["loss"], want["loss"], 1e-5) and within(got["d_fcn"], want["d_fcn"], 2e-5)
    c["seg_gt"][(c["seg_gt"] != 255) & (c["seg_gt"] >= 7)] = 255     # the same pixels ignored instead
    again = run_sem(c)
    assert again["loss"] == got["loss"] and np.array_equal(again["d_fcn"], got["d_fcn"])


def test_semantic_label_dtypes_give_the_same_bytes():
    c = TL.semantic_case(24, 19, 33, 45, (7, 5), 0.1, 0.01)
    a, b = run_sem(c, seg_dtype=torch.uint8), run_sem(c, seg_dtype=torch.int64)
    assert torch.equal(a["raw"][0], b["raw"][0]) and torch.equal(a["raw"][1], b["raw"][1])


# ---- RPN loss ---------------------------------------------------------------------------------
def rpn_targets_case(seed=31):
    """RPNTargets for a 1024 x 2048 image (fields 512 x 512 at stride 4, larger than the 256 x 512 map), numpy."""
    from upsnet_b200.training import RPNTargets
    rng = np.random.default_rng(seed)
    xy = rng.uniform(0, [1900, 950], (30, 2))
    wh = rng.uniform(16, 300, (30, 2))
    gt = np.concatenate([xy, np.minimum(xy + wh, [2047, 1023])], 1).astype(np.float32)
    lab = RPNTargets(max_size=2048)(t(gt), 1024, 2048, seed=seed)
    c = {"label": {k: v.cpu().numpy() for k, v in lab.items()}, "scores": [], "preds": []}
    for s in TL.STRIDES:
        h, w = -(-1024 // s), -(-2048 // s)
        c["scores"].append((rng.standard_normal((1, 3, h, w)) * 2).astype(np.float32))
        c["preds"].append((rng.standard_normal((1, 12, h, w)) * 0.3).astype(np.float32))
    return c, lab


def test_rpn_on_rpn_targets_vs_oracle():
    c, lab = rpn_targets_case()
    assert lab["rpn_labels_fpn4"].shape[2] > c["scores"][0].shape[2]
    from upsnet_b200 import RPNLoss
    xs = [t(a).requires_grad_(True) for a in c["scores"]]
    ps = [t(a).requires_grad_(True) for a in c["preds"]]
    cls_loss, bbox_loss = RPNLoss(rpn_batch_size=256)(xs, ps, lab)        # the views RPNTargets returns, read in place
    (cls_loss + bbox_loss).backward()
    want = TL.rpn(c, 256)
    assert rel_ok(cls_loss.detach(), want["cls_loss"], 1e-5) and rel_ok(bbox_loss.detach(), want["bbox_loss"], 1e-5)
    for x, p, ds, dp in zip(xs, ps, want["d_scores"], want["d_preds"]):
        assert within(x.grad.cpu().numpy(), ds, 1e-5) and within(p.grad.cpu().numpy(), dp, 1e-5)


def test_rpn_config_and_grad_out_scaling():
    from upsnet_b200 import RPNLoss

    class Cfg:
        class train:
            rpn_batch_size, batch_size = 128, 1
    assert RPNLoss(Cfg).rpn_batch_size == 128
    c = rpn_fixture("fields_larger")
    got, want = run_rpn(c, 128, go=(2.5, -0.5)), TL.rpn(c, 128)
    for g, w_ in zip(got["d_scores"], want["d_scores"]):
        assert within(g, 2.5 * w_, 1e-5)
    for g, w_ in zip(got["d_preds"], want["d_preds"]):
        assert within(g, -0.5 * w_, 1e-5)


# ---- Mask R-CNN loss --------------------------------------------------------------------------
def proposal_case(seed=41):
    import proposal_target_oracle as PT
    from upsnet_b200.training import ProposalTargets
    rng = np.random.default_rng(seed)
    e = PT.random_entry(rng, 600, 1000, 20, 81)
    rois = PT.random_rois(rng, e, 2000, 600, 1000, 800 / 600)
    out = ProposalTargets(num_classes=81, batch_rois=512).from_roidb(t(rois), e, np.array([[800, 1333, 800 / 600]],
                                                                                          np.float32), seed=seed)
    rois_, labels, bt, biw, bow, mask_rois, mask_int32 = out[:7]
    R, n = labels.shape[0], mask_rois.shape[0]
    c = dict(cls_score=(rng.standard_normal((R, 81)) * 2).astype(np.float32),
             bbox_pred=(rng.standard_normal((R, 324)) * 0.8).astype(np.float32),
             mask_score=(rng.standard_normal((n, 81, 28, 28)) * 3).astype(np.float32),
             cls_label=labels.cpu().numpy(), bbox_target=bt.cpu().numpy(), bbox_inside_weight=biw.cpu().numpy(),
             bbox_outside_weight=bow.cpu().numpy(), mask_target=mask_int32.cpu().numpy())
    return c, (labels, bt, biw, bow, mask_int32)


def test_mask_rcnn_on_proposal_targets_vs_oracle():
    from upsnet_b200 import MaskRCNNLoss
    c, (labels, bt, biw, bow, mask_int32) = proposal_case()
    assert mask_int32.shape[1] == 81 * 28 * 28 and mask_int32.shape[0] >= 16
    x, p, ms = (t(c[k]).requires_grad_(True) for k in ("cls_score", "bbox_pred", "mask_score"))
    m = MaskRCNNLoss()
    cls_loss, bbox_loss, mask_loss, acc = m(x, p, ms, labels, bt, biw, bow, mask_int32)   # ProposalTargets' outputs as they are
    (cls_loss + bbox_loss + mask_loss).backward()
    valid, ignored, matches, mw = m.counts.cpu().tolist()
    got = dict(cls_loss=float(cls_loss.detach()), bbox_loss=float(bbox_loss.detach()), mask_loss=float(mask_loss.detach()),
               accuracy=float(acc), valid=valid, ignored=ignored, matches=matches, mask_weight=mw,
               d_cls=x.grad.cpu().numpy(), d_bbox=p.grad.cpu().numpy(), d_mask=ms.grad.cpu().numpy())
    check_mrcnn(got, TL.mask_rcnn(c))


def test_mask_rcnn_ignored_rows_and_no_mask_target():
    c = TL.mask_rcnn_case(42, 128, 81, 40, 28, 0.3)
    got, want = run_mrcnn(c), TL.mask_rcnn(c)
    assert want["ignored"] > 0 and want["accuracy"] < 0
    check_mrcnn(got, want)
    c = TL.mask_rcnn_case(43, 64, 81, 20, 28, 0.0, True)
    got = run_mrcnn(c)
    assert got["mask_loss"] == 0.0 and got["mask_weight"] == 0 and not got["d_mask"].any()
    c = TL.mask_rcnn_case(44, 16, 9, 4)
    c["cls_label"][3] = 9                     # neither -1 nor a class: no loss, no gradient, never correct
    got, want = run_mrcnn(c), TL.mask_rcnn(c)
    check_mrcnn(got, want)
    assert not got["d_cls"][3].any()


def test_mask_rcnn_grad_out_scaling():
    c = TL.mask_rcnn_case(45, 64, 81, 16)
    got, want = run_mrcnn(c, go=(3.0, 0.25, -2.0)), TL.mask_rcnn(c)
    assert within(got["d_cls"], 3.0 * want["d_cls"], 1e-5)
    assert within(got["d_bbox"], 0.25 * want["d_bbox"], 1e-5)
    assert within(got["d_mask"], -2.0 * want["d_mask"], 1e-5)


# ---- drop-in: the modules vs the unfused fp32 composition on the device ------------------------
def test_drop_in_against_the_unfused_composition():
    c = TL.semantic_case(51, 19, 64, 96, (12, 20), 0.1)
    got, want = run_sem(c), TL.semantic(c, torch.float32, DEV)
    assert rel_ok(got["loss"], want["loss"], 1e-5) and within(got["d_fcn"], want["d_fcn"], 2e-5)
    c = rpn_fixture("fields_larger")
    got, want = run_rpn(c), TL.rpn(c, 256, torch.float32, DEV)
    assert rel_ok(got["cls_loss"], want["cls_loss"], 1e-5) and rel_ok(got["bbox_loss"], want["bbox_loss"], 1e-5)
    for a, b in zip(got["d_scores"] + got["d_preds"], want["d_scores"] + want["d_preds"]):
        assert within(a, b, 1e-5)
    c = TL.mask_rcnn_case(52, 128, 81, 32)
    check_mrcnn(run_mrcnn(c), TL.mask_rcnn(c, torch.float32, DEV))


def test_semantic_grad_out_scaling():
    c = TL.semantic_case(53, 19, 24, 40, (8, 8))
    one, three = run_sem(c), run_sem(c, grad_out=3.0)
    assert within(three["d_fcn"], 3.0 * one["d_fcn"], 1e-6)


# ---- determinism ------------------------------------------------------------------------------
def test_same_bytes_side_stream_and_graph_replay():
    from upsnet_b200 import MaskRCNNLoss, RPNLoss, SemanticLoss
    cs = TL.semantic_case(61, 19, 64, 128, (16, 16), 0.1)
    x, seg = t(cs["fcn"]).requires_grad_(True), t(cs["seg_gt"])
    xs, ps, lab = rpn_device(rpn_fixture("fields_larger"))
    cm = TL.mask_rcnn_case(62, 128, 81, 32)
    mi = [t(cm[k]) for k in TL.NAMES]
    for i in range(3):
        mi[i].requires_grad_(True)
    sem, rpn, mr = SemanticLoss(), RPNLoss(), MaskRCNNLoss()
    leaves = [x] + xs + ps + mi[:3]

    def call():
        for v in leaves:
            v.grad = None
        ls = sem(x, seg)
        a, b = rpn(xs, ps, lab)
        m = mr(*mi)
        (ls + a + b + m[0] + m[1] + m[2]).backward()
        return [ls.detach(), a.detach(), b.detach()] + [v.detach() for v in m] + [sem.counts, mr.counts] + \
            [v.grad for v in leaves]

    ref = [v.clone() for v in call()]
    for u, v in zip(ref, call()):
        assert torch.equal(u, v) or (u.is_floating_point() and torch.equal(u.isnan(), v.isnan()))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        b = [v.clone() for v in call()]
    torch.cuda.current_stream().wait_stream(side)
    for u, v in zip(ref, b):
        assert torch.equal(u, v)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g = call()
    for v in g:
        v.fill_(7)
    graph.replay()
    torch.cuda.synchronize()
    for u, v in zip(ref, g):
        assert torch.equal(u, v)


# ---- errors -----------------------------------------------------------------------------------
def test_errors():
    from upsnet_b200 import MaskRCNNLoss, RPNLoss, SemanticLoss
    from upsnet_b200._lib import UpsnetError
    c = TL.semantic_case(71, 5, 8, 8)
    x, seg = t(c["fcn"]), t(c["seg_gt"])
    with pytest.raises(UpsnetError):
        SemanticLoss()(x.cpu(), seg.cpu())
    with pytest.raises(UpsnetError):
        SemanticLoss()(x, seg[:, :-4])                          # not 4h x 4w
    with pytest.raises(UpsnetError):
        SemanticLoss()(x.expand(2, -1, -1, -1), seg)           # batch 2
    with pytest.raises(UpsnetError):
        SemanticLoss()(x, seg.float())
    xs, ps, lab = rpn_device(rpn_fixture("fields_larger"))
    with pytest.raises(UpsnetError):
        RPNLoss()([v.cpu() for v in xs], [v.cpu() for v in ps], lab)
    with pytest.raises(UpsnetError):
        RPNLoss()(xs, ps[:-1], lab)
    with pytest.raises(UpsnetError):
        RPNLoss()([v.expand(2, -1, -1, -1) for v in xs], [v.expand(2, -1, -1, -1) for v in ps], lab)
    small = dict(lab, rpn_labels_fpn4=lab["rpn_labels_fpn4"][:, :, :xs[0].shape[2] - 1])
    with pytest.raises(UpsnetError):
        RPNLoss()(xs, ps, small)                               # a field smaller than the map
    with pytest.raises(UpsnetError):
        RPNLoss()(xs, ps, {k: v for k, v in lab.items() if not k.endswith("fpn16")})
    cm = TL.mask_rcnn_case(72, 16, 9, 4)
    mi = [t(cm[k]) for k in TL.NAMES]
    with pytest.raises(UpsnetError):
        MaskRCNNLoss()(*[v.cpu() for v in mi])
    with pytest.raises(UpsnetError):
        MaskRCNNLoss()(*mi[:3], mi[3][:-1], *mi[4:])
    with pytest.raises(UpsnetError):
        MaskRCNNLoss()(*mi[:4], mi[4][:, :-4], *mi[5:])
    with pytest.raises(UpsnetError):
        MaskRCNNLoss()(*mi[:7], mi[7][:, :-1])
