"""The fused panoptic loss on the device (csrc/panoptic_loss.cu through upsnet_b200.training.PanopticLoss) against the
reference fixtures (tests/golden/reference_panoptic_loss.npz), the fp64 oracle (tests/panoptic_loss_oracle.py) and the
unfused composition of this package's own SegTerm / MaskTerm / MaskMatching with F.cross_entropy and autograd."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import panoptic_loss_oracle as PL  # noqa: E402
from test_panoptic_loss_cpu import CASES, Z, fixture_case  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def module_for(c):
    from upsnet_b200.training import PanopticLoss
    return PanopticLoss(num_seg_classes=c["fcn"].shape[1], num_classes=c["num_classes"], enable_void=c["enable_void"])


def device_inputs(c, C_=None, mask_dtype=torch.uint8):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)  # noqa: E731
    ms = c["mask_score"] if C_ != 1 else PL.selected(c)[:, None].numpy()
    keep = None if c["keep"] is None else t(c["keep"])
    return (t(c["fcn"]).requires_grad_(True), t(ms).requires_grad_(True), t(c["rois"]), t(c["cls"]), t(c["seg_gt"]),
            t(c["mask_gt"]).to(mask_dtype), keep)


def run(c, grad_out=None, C_=None, mask_dtype=torch.uint8):
    """-> dict like the oracle's: loss, accuracy, correct, ignored, d_fcn, d_mask (selected channels), d_mask_full."""
    m = module_for(c)
    inp = device_inputs(c, C_, mask_dtype)
    loss, acc = m(*inp)
    (loss if grad_out is None else loss * grad_out).backward()
    fcn, ms = inp[0], inp[1]
    k = ms.shape[0]
    full = ms.grad.cpu().numpy()
    sel = full[np.arange(k), c["cls"] if ms.shape[1] > 1 else 0]
    correct, ignored = (int(v) for v in m.counts.cpu())
    return dict(loss=float(loss.detach()), accuracy=float(acc), correct=correct, ignored=ignored,
                d_fcn=fcn.grad.cpu().numpy(), d_mask=sel, d_mask_full=full, loss_t=loss.detach(), acc_t=acc)


def within(got, want, rel):
    return np.abs(got - want).max() <= rel * np.abs(want).max()


@pytest.mark.parametrize("name", CASES)
def test_fixture(name):
    p = name + "/"
    c = fixture_case(name)
    m = module_for(c)
    inp = device_inputs(c)
    assert np.array_equal(m.panoptic_gt(inp[4], inp[5], inp[6]).cpu().numpy(), Z[p + "gt"])
    got = run(c)
    assert abs(got["loss"] - float(Z[p + "loss"])) <= 1e-5 * abs(float(Z[p + "loss"]))
    assert got["correct"] == int(Z[p + "correct"]) and got["ignored"] == int(Z[p + "ignored"])
    assert abs(got["accuracy"] - float(Z[p + "accuracy"])) <= 1e-6
    assert within(got["d_fcn"], Z[p + "d_fcn"], 1e-5)
    assert within(got["d_mask"], Z[p + "d_mask"], 1e-5)


@pytest.mark.parametrize("name", ["cityscapes", "coco_k63"])
def test_full_size_against_fp64_oracle(name):
    c = PL.case(PL.FULL[name])
    want = PL.run(c, torch.float64)
    got = run(c)
    assert abs(got["loss"] - want["loss"]) <= 1e-5 * abs(want["loss"])
    assert within(got["d_fcn"], want["d_fcn"], 2e-5)
    assert within(got["d_mask"], want["d_mask"], 2e-5)
    k = len(c["cls"])
    rest = got["d_mask_full"].copy()
    rest[np.arange(k), c["cls"]] = 0
    assert not rest.any()
    assert not got["d_fcn"][:, :, want["gt"][0] == 255].any()
    assert got["ignored"] == want["ignored"]
    # the arg-max of the pixels whose fp64 top-two margin is below 1e-4 may differ in float32: set them aside
    close_call = int((want["margin"] < 1e-4).sum())
    print("%s: %d of %d pixels with a top-two margin below 1e-4" % (name, close_call, want["margin"].size))
    assert abs(got["correct"] - want["correct"]) <= close_call


def unfused(c, inp):
    """What a user of this package writes without the fused op: resnet_upsnet.py:156-179, 250-257 on the three modules."""
    from upsnet_b200 import MaskMatching, MaskTerm, SegTerm
    fcn, ms, rois, cls, seg, mgt, keep = inp
    S, nc, void = fcn.shape[1], c["num_classes"], c["enable_void"]
    sel = ms.gather(1, cls.view(-1, 1, 1, 1).expand(-1, -1, 28, 28))
    seg_logits, seg_inst = SegTerm(S, num_classes=nc)(cls, fcn, rois)
    mask_logits = MaskTerm(S, num_classes=nc)(sel, rois, cls, fcn)
    parts = [seg_logits, seg_inst + mask_logits]
    if void:
        parts.append(fcn[:, S - nc + 1:].max(1, keepdim=True)[0] - seg_inst.max(1, keepdim=True)[0])
    logits = torch.cat(parts, 1)
    with torch.no_grad():
        gt = MaskMatching(S, void, num_classes=nc)(seg, mgt.long(), keep)
    loss = torch.nn.functional.cross_entropy(logits, gt, ignore_index=255, reduction="none").mean()
    correct = (logits.detach().max(1)[1].view(-1) == gt.view(-1)).sum()
    return loss, correct, (gt == 255).sum(), logits.detach()


@pytest.mark.parametrize("name", ["cityscapes", "coco_k10"])
def test_drop_in_for_the_unfused_composition(name):
    c = PL.case(PL.FULL[name])
    got = run(c)
    inp = device_inputs(c)
    loss, correct, ignored, logits = unfused(c, inp)
    loss.backward()
    k, loss = len(c["cls"]), float(loss.detach())
    assert abs(got["loss"] - loss) <= 1e-5 * abs(loss)
    assert within(got["d_fcn"], inp[0].grad.cpu().numpy(), 2e-5)
    assert within(got["d_mask_full"], inp[1].grad.cpu().numpy(), 2e-5)
    assert got["ignored"] == int(ignored)
    top2 = logits.topk(2, dim=1)[0][0]
    assert abs(got["correct"] - int(correct)) <= int(((top2[0] - top2[1]) < 1e-4).sum())
    assert k == inp[1].shape[0]


def test_grad_out_scaling_and_gathered_mask_score():
    c = PL.case(PL.SMALL["coco_void"])
    one, three = run(c), run(c, grad_out=3.0)
    assert one["loss"] == three["loss"]
    assert within(three["d_fcn"], 3 * one["d_fcn"], 1e-6) and within(three["d_mask"], 3 * one["d_mask"], 1e-6)
    gathered = run(c, C_=1)
    assert gathered["loss"] == one["loss"] and gathered["correct"] == one["correct"]
    assert np.array_equal(gathered["d_mask"], one["d_mask"]) and np.array_equal(gathered["d_fcn"], one["d_fcn"])
    want = PL.run(c, torch.float64, grad_out=3.0, C=1)
    assert within(three["d_mask"], want["d_mask"], 2e-5)


def test_same_bytes_side_stream_and_graph_replay():
    c = PL.case(PL.FULL["coco_k10"])
    m = module_for(c)
    inp = device_inputs(c)

    def call():
        for t in inp[:2]:
            t.grad = None
        loss, acc = m(*inp)
        loss.backward()
        return [loss.detach(), acc, m.counts, inp[0].grad, inp[1].grad]

    a = [t.clone() for t in call()]
    for x, y in zip(a, call()):
        assert torch.equal(x, y)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        b = [t.clone() for t in call()]
    torch.cuda.current_stream().wait_stream(side)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g = call()
    for t in g:
        t.fill_(7)
    graph.replay()
    torch.cuda.synchronize()
    for x, y in zip(a, g):
        assert torch.equal(x, y)


def test_mask_gt_dtypes_and_the_branch_without_void():
    for name in ("cityscapes_void", "no_void"):
        c = PL.case(PL.SMALL[name])
        a, b = run(c, mask_dtype=torch.uint8), run(c, mask_dtype=torch.int64)
        for key in ("loss", "correct", "ignored"):
            assert a[key] == b[key]
        assert np.array_equal(a["d_fcn"], b["d_fcn"]) and np.array_equal(a["d_mask_full"], b["d_mask_full"])
    c = PL.case(PL.SMALL["no_void"])
    assert c["keep"] is None and not c["enable_void"]
    want, got = PL.run(c, torch.float64), run(c)
    assert abs(got["loss"] - want["loss"]) <= 1e-5 * abs(want["loss"])
    assert got["ignored"] == want["ignored"] and abs(got["correct"] - want["correct"]) <= int((want["margin"] < 1e-4).sum())
    assert within(got["d_fcn"], want["d_fcn"], 2e-5) and within(got["d_mask"], want["d_mask"], 2e-5)
    m = module_for(c)
    inp = device_inputs(c)
    for mg in (inp[5], inp[5].long()):
        assert np.array_equal(m.panoptic_gt(inp[4], mg).cpu().numpy(), want["gt"])


def test_draw_key_on_the_device_equals_the_host_rule():
    from upsnet_b200._lib import check, lib, ptr, stream_ptr
    from upsnet_b200.training import draw_keys
    for seed in (0, 9, 2 ** 63 + 11):
        out = torch.empty(1000, dtype=torch.int64, device=DEV)
        check(lib().upsnet_draw_keys(C.c_ulonglong(seed), 0, 1000, ptr(out), stream_ptr(DEV)), "draw_keys")
        assert np.array_equal(out.cpu().numpy().view(np.uint64), draw_keys(seed, 1000))


def test_errors():
    from upsnet_b200._lib import UpsnetError
    from upsnet_b200.training import PanopticLoss
    c = PL.case(PL.SMALL["cityscapes_void"])
    m = module_for(c)
    fcn, ms, rois, cls, seg, mgt, keep = (t.detach() if t is not None else None for t in device_inputs(c))
    bad = [
        (fcn, ms[:0], rois[:0], cls[:0], seg, mgt, keep[:0]),                   # k == 0
        (fcn.cpu(), ms, rois, cls, seg, mgt, keep),                             # CPU tensors
        (fcn, ms, rois, cls, seg.cpu(), mgt, keep),
        (fcn.repeat(2, 1, 1, 1), ms, rois, cls, seg, mgt, keep),                # batch 2
        (fcn[:, :-1], ms, rois, cls, seg, mgt, keep),                           # shape mismatches
        (fcn, ms[:, :3], rois, cls, seg, mgt, keep),
        (fcn, ms[:, :, :14], rois, cls, seg, mgt, keep),
        (fcn, ms, rois[:-1], cls, seg, mgt, keep),
        (fcn, ms, rois, cls[:-1], seg, mgt, keep),
        (fcn, ms, rois, cls, seg[:, :-1], mgt[:, :-1], keep),
        (fcn, ms, rois, cls, seg, mgt[:, :, :-1], keep),
        (fcn, ms, rois, cls, seg, mgt, keep[:-1]),
        (fcn, ms, rois, cls, seg, mgt.float(), keep),
        (fcn, ms, rois, cls, seg, mgt, np.array([0, 1, 99] + [2] * (len(cls) - 3))),   # keep_inds outside mask_gt
        (fcn, ms, rois, cls, seg, mgt, None),                                   # enable_void without keep_inds
    ]
    for args in bad:
        with pytest.raises(UpsnetError):
            m(*args)
    no_void = PanopticLoss(num_seg_classes=19, num_classes=9, enable_void=False)
    with pytest.raises(UpsnetError):
        no_void(fcn, ms, rois, cls, seg, mgt, keep)                             # keep_inds without enable_void
    with pytest.raises(UpsnetError):
        no_void(fcn, ms, rois, cls, seg, mgt)                                   # all of mask_gt, but G != k
    with pytest.raises(UpsnetError):
        PanopticLoss()
    torch.cuda.synchronize()
