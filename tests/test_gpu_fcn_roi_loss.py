"""The fused FCN ROI loss on the device (csrc/train_loss.cu through upsnet_b200.training.FcnRoiLoss) against the
float64 oracle (tests/fcn_roi_loss_oracle.py) and the reference fixture (tests/golden/reference_fcn_roi_loss.npz), and
training.linear at one row.

Gradient bound: every element of d fcn_score and d bias is held to C_GRAD * sum of |terms|, the terms being tap weight
* (softmax + onehot) * |grad_out| / (R*M*M) of every cell that reaches it (oracle.grad_bounds).  The float32 kernel
differs from float64 by rounding in the roi scores (a sum of 16 products), the log-sum-exp over S channels and the
softmax, each a few ulp relative to the logits' scale, amplified by the exponent: C_GRAD = 1e-4 (the sample weights
themselves are bit-identical, the oracle computes the coordinates with the kernels' float32 roundings).  Measured worst
ratio on an H100 80GB HBM3 at 700 W: 3.8e-6 (d fcn_score), 4.4e-7 (d bias)."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import fcn_roi_loss_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
C_GRAD = 1e-4
LOSS_REL = 2e-6
Z_PATH = os.path.join(HERE, "golden", "reference_fcn_roi_loss.npz")


def device_case(name):
    c = O.case(name)
    feat = O.feat_of([t.to(DEV) for t in c["levels"]])
    fcn = torch.nn.functional.conv2d(feat, c["weight"].double().to(DEV), c["bias"].double().to(DEV)).float()
    return fcn, c["bias"].to(DEV), c["rois"].to(DEV), c["seg"].to(DEV), c, feat


def random_case(seed, S, R, h, w):
    g = torch.Generator().manual_seed(seed)
    fcn = (torch.randn(1, S, h, w, generator=g) * 3).to(DEV)
    bias = torch.randn(S, generator=g).to(DEV)
    rois = O.boxes(g, R, h, w, "random").to(DEV)
    seg = torch.randint(0, S, (R, O.M, O.M), generator=g)
    seg[torch.rand(R, O.M, O.M, generator=g) < 0.2] = 255
    return fcn, bias, rois, seg.to(DEV)


def run(fcn, bias, rois, seg, grad_out=1.0):
    from upsnet_b200 import FcnRoiLoss
    m = FcnRoiLoss(28)
    x, b = fcn.clone().requires_grad_(True), bias.clone().requires_grad_(True)
    loss = m(x, b, rois, seg)
    (loss * grad_out).backward()
    return loss.detach(), x.grad, b.grad, m.counts


def check_against_oracle(fcn, bias, rois, seg, grad_out=1.0, label=""):
    loss, dx, db, counts = run(fcn, bias, rois, seg, grad_out)
    x64, b64 = fcn[0].double().requires_grad_(True), bias.double().requires_grad_(True)
    want = O.loss_from_score(x64, b64, rois, seg)
    (want * grad_out).backward()
    want = want.detach()
    assert abs(float(loss) - float(want)) <= LOSS_REL * abs(float(want)), (float(loss), float(want))
    bx, bb = O.grad_bounds(fcn[0], bias, rois, seg, grad_out=grad_out)
    ex = (dx[0].double() - x64.grad).abs()
    eb = (db.double() - b64.grad).abs()
    rx = float((ex / bx.clamp_min(1e-300)).max())
    rb = float((eb / bb.clamp_min(1e-300)).max())
    print("%s worst |err| / sum|terms|: d fcn_score %.3g, d bias %.3g (C_GRAD %g)" % (label, rx, rb, C_GRAD))
    assert bool((ex <= C_GRAD * bx).all()) and bool((eb <= C_GRAD * bb).all())
    valid = ((seg >= 0) & (seg < fcn.shape[1])).sum()
    assert counts.tolist() == [int(valid), 0]
    return loss, dx, db


@pytest.mark.parametrize("name", sorted(O.CASES))
def test_fixture_cases_against_oracle_and_reference(name):
    fcn, bias, rois, seg, c, feat = device_case(name)
    loss, dx, db = check_against_oracle(fcn, bias, rois, seg, label=name)
    Z = np.load(Z_PATH)
    p = "case/%s/" % name
    assert O.inputs_digest(c) == str(Z[p + "inputs_sha256"])
    assert abs(float(loss) - float(Z[p + "loss"])) <= 1e-5 * abs(float(Z[p + "loss"]))
    # the reference's score-conv gradients, by the chain rule through fcn_score = W feat + b
    dW = torch.einsum("syx,cyx->sc", dx[0].double(), feat[0]).cpu().numpy()
    dB = (dx[0].double().sum((1, 2)) + db.double()).cpu().numpy()
    scale = np.abs(Z[p + "d_weight"]).max()
    assert np.abs(dW - Z[p + "d_weight"].reshape(dW.shape)).max() <= 1e-4 * scale
    assert np.abs(dB - Z[p + "d_bias"]).max() <= 1e-4 * np.abs(Z[p + "d_bias"]).max()


def test_coco_size_r90_and_adjoint():
    fcn, bias, rois, seg = random_case(5, 133, 90, 200, 336)
    loss, dx, db = check_against_oracle(fcn, bias, rois, seg, label="coco r90")
    # adjoint identity: <d fcn_score, v> equals the directional derivative of the oracle along v
    v = torch.randn_like(fcn[0], dtype=torch.float64)
    x64 = fcn[0].double().requires_grad_(True)
    O.loss_from_score(x64, bias, rois, seg).backward()
    lhs, rhs = float((dx[0].double() * v).sum()), float((x64.grad * v).sum())
    assert abs(lhs - rhs) <= 1e-5 * float((x64.grad.abs() * v.abs()).sum())
    # d fcn_score is written everywhere: zero away from every roi
    By, Bx, _ = O.roi_align_weights(rois, 200, 336)
    far = (By.sum((0, 1))[:, None] * Bx.sum((0, 1))[None, :]) == 0
    assert bool((dx[0][:, far] == 0).all())


def test_grad_out_scaling_and_uint8_targets():
    fcn, bias, rois, seg = random_case(6, 19, 12, 32, 48)
    check_against_oracle(fcn, bias, rois, seg, grad_out=-3.0, label="grad_out -3")
    l8, dx8, db8, c8 = run(fcn, bias, rois, seg.to(torch.uint8))
    l64, dx64, db64, c64 = run(fcn, bias, rois, seg)
    assert torch.equal(l8, l64) and torch.equal(dx8, dx64) and torch.equal(db8, db64) and torch.equal(c8, c64)


def test_invalid_targets_are_counted_and_give_nothing():
    fcn, bias, rois, seg = random_case(7, 19, 4, 16, 24)
    bad = seg.clone()
    bad[0, :5, :] = 40                                   # neither 255 nor a class
    ign = seg.clone()
    ign[0, :5, :] = 255
    lb, dxb, dbb, cb = run(fcn, bias, rois, bad)
    li, dxi, dbi, ci = run(fcn, bias, rois, ign)
    assert cb.tolist() == [int(ci[0]), 5 * 28]
    assert torch.equal(lb, li) and torch.equal(dxb, dxi) and torch.equal(dbb, dbi)


def test_same_bytes_side_stream_and_graph_replay():
    from upsnet_b200 import FcnRoiLoss
    fcn, bias, rois, seg = random_case(8, 133, 30, 64, 96)
    x, b = fcn.clone().requires_grad_(True), bias.clone().requires_grad_(True)
    m = FcnRoiLoss(28)

    def call():
        x.grad = b.grad = None
        loss = m(x, b, rois, seg)
        loss.backward()
        return [loss.detach(), m.counts, x.grad, b.grad]

    ref = [v.clone() for v in call()]
    for u, v in zip(ref, call()):
        assert torch.equal(u, v)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        s = [v.clone() for v in call()]
    torch.cuda.current_stream().wait_stream(side)
    for u, v in zip(ref, s):
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


def test_peak_memory_at_coco_size():
    from upsnet_b200 import FcnRoiLoss
    fcn, bias, rois, seg = random_case(9, 133, 90, 200, 336)
    x, b = fcn.clone().requires_grad_(True), bias.clone().requires_grad_(True)
    FcnRoiLoss(28)(x, b, rois, seg).backward()          # builds the library and the allocator pools first
    x.grad = b.grad = None
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    FcnRoiLoss(28)(x, b, rois, seg).backward()
    torch.cuda.synchronize()
    grew = torch.cuda.max_memory_allocated() - base - x.numel() * 4    # d fcn_score itself is an output
    print("peak above inputs and d fcn_score: %.1f MB" % (grew / 2 ** 20))
    assert grew < 48 * 2 ** 20


def test_unsupported_shapes():
    from upsnet_b200 import FcnRoiLoss
    from upsnet_b200._lib import E_UNSUPPORTED, UpsnetError, query_bytes, try_call
    fcn, bias, rois, seg = random_case(10, 19, 4, 16, 24)
    with pytest.raises(UpsnetError, match="unsupported"):
        FcnRoiLoss(28)(fcn, bias, rois[:0], seg[:0])
    many = rois[:1].repeat(1025, 1)
    with pytest.raises(UpsnetError, match="unsupported"):
        FcnRoiLoss(28)(fcn, bias, many, seg[:1].repeat(1025, 1, 1))
    with pytest.raises(UpsnetError, match="unsupported"):
        FcnRoiLoss(96)(fcn, bias, rois, torch.zeros(4, 96, 96, dtype=torch.int64, device=DEV))
    with pytest.raises(UpsnetError, match="seg_roi_gt"):
        FcnRoiLoss(28)(fcn, bias, rois, seg[:3])
    # S*h*w >= 2^31 and sampling_ratio 3: refused by the entry point before it reads or launches anything
    loss, counts = torch.empty((), device=DEV), torch.empty(2, dtype=torch.int32, device=DEV)
    lse = torch.empty(4 * 28 * 28, device=DEV)
    ws = torch.empty(query_bytes("fcn_roi_loss_workspace_bytes", 20000, 4, 28, 0), dtype=torch.uint8, device=DEV)
    for S, h, w, sr in ((20000, 330, 330, 2), (19, 16, 24, 3)):
        rc = try_call("fcn_roi_loss_forward", DEV, fcn, bias, S, h, w, rois, 4, seg, 1, 28, sr, 0.25, loss, counts, lse,
                      ws, ws.numel())
        assert rc == E_UNSUPPORTED
    assert query_bytes("fcn_roi_loss_workspace_bytes", 133, 90, 28, 1) >= 133 * 90 * 784 * 4


@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_linear_one_row(prec):
    from upsnet_b200 import training
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 2048, generator=g).to(DEV).requires_grad_(True)
    w = (torch.randn(256, 2048, generator=g) * 0.02).to(DEV).requires_grad_(True)
    b = torch.randn(256, generator=g).to(DEV).requires_grad_(True)
    gy = torch.randn(1, 256, generator=g).to(DEV)
    y = training.linear(x, w, b, precision=prec)
    y.backward(gy)
    x64, w64, b64 = (t.detach().double().requires_grad_(True) for t in (x, w, b))
    y64 = x64 @ w64.t() + b64
    y64.backward(gy.double())
    c = 1e-4 if prec == "bf16x3" else 3e-2       # bf16x3: ~2^-16 per product; bf16: ~2^-8 per operand
    ay = x64.detach().abs() @ w64.detach().abs().t() + b64.detach().abs()
    ax = gy.double().abs() @ w64.detach().abs()
    aw = gy.double().abs().t() @ x64.detach().abs()
    for got, want, bound, what in ((y, y64, ay, "y"), (x.grad, x64.grad, ax, "dx"), (w.grad, w64.grad, aw, "dw"),
                                   (b.grad, b64.grad, gy.double().abs()[0], "db")):
        r = float(((got.double() - want).abs() / bound.clamp_min(1e-300)).max())
        print("linear R=1 %s %s worst ratio %.3g" % (prec, what, r))
        assert r <= c
