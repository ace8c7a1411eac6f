"""The training forward of resnet_upsnet on the device (forward(data, label)) against the float64 oracle of
tests/train_forward_oracle.py, and the adjoint kernel of the semantic head's level sum (upsnet_fcn_score_fuse_backward)
against float64 autograd."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import train_forward_oracle as TF  # noqa: E402
from sgd_oracle import OracleSGD  # noqa: E402

pytestmark = pytest.mark.gpu


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


# ------------------------------------------------------------------------------------------------
# upsnet_fcn_score_fuse_backward
# ------------------------------------------------------------------------------------------------
def _fuse64(s):
    return s[0] + sum(F.interpolate(t, None, 2 ** l, mode="bilinear", align_corners=False) for l, t in enumerate(s[1:], 1))


@pytest.mark.parametrize("P,H,W", [(1, 8, 8), (3, 24, 40), (19, 72, 136), (2, 256, 512)])
def test_fuse_backward_vs_autograd(dev, P, H, W):
    from upsnet_b200.training import fcn_score_fuse_backward
    g = torch.Generator().manual_seed(H * W + P)
    d = torch.randn(1, P, H, W, generator=g).to(dev)
    got = fcn_score_fuse_backward(d)
    s = [torch.zeros(1, P, H >> l, W >> l, dtype=torch.float64, device=dev, requires_grad=True) for l in range(4)]
    want = torch.autograd.grad(_fuse64(s), s, d.double())
    mag = torch.autograd.grad(_fuse64(s), s, d.double().abs())          # sum of |terms| of every element
    c = 32 * 2.0 ** -24
    for l in range(1, 4):
        err = (got[l - 1].double() - want[l]).abs()
        assert got[l - 1].shape == want[l].shape
        assert bool((err <= c * mag[l] + 1e-30).all()), (l, float((err / (mag[l] + 1e-30)).max()))
    # the adjoint identity <fuse(s), d> = <s, fuse^T(d)> (fuse on the device, in float32)
    from upsnet_b200 import operators as ops
    s32 = [torch.randn(1, P, H >> l, W >> l, generator=g).to(dev) for l in range(4)]
    lhs = (ops.fcn_score_fuse(*s32).double() * d.double()).sum()
    rhs = (s32[0].double() * d.double()).sum() + sum((s32[l].double() * got[l - 1].double()).sum() for l in range(1, 4))
    scale = float((_fuse64([t.double().abs() for t in s32]) * d.double().abs()).sum())
    assert abs(float(lhs - rhs)) <= 1e-5 * scale
    again = fcn_score_fuse_backward(d)
    assert all(torch.equal(a, b) for a, b in zip(got, again))


def test_fuse_backward_rejects_bad_shapes(dev):
    from upsnet_b200._lib import UpsnetError
    from upsnet_b200.training import fcn_score_fuse_backward
    with pytest.raises(UpsnetError):
        fcn_score_fuse_backward(torch.zeros(1, 2, 12, 16, device=dev))
    with pytest.raises(UpsnetError):
        fcn_score_fuse_backward(torch.zeros(1, 2, 16, 20, device=dev))


# ------------------------------------------------------------------------------------------------
# the training forward
# ------------------------------------------------------------------------------------------------
def _setup(dev, dconv=100, H=256, W=512, G=8, seed=0, depth=(2, 2, 2, 2)):
    from upsnet_b200.model import UPSNetConfig
    from upsnet_b200.synthetic import synthetic_model
    from upsnet_b200.training import PanopticLabels, RPNTargets
    m = synthetic_model(UPSNetConfig(backbone_with_dconv=dconv), depth=depth, seed=seed, device=dev)
    entry, lmap = TF.synthetic_entry(seed + 1, H, W, G)
    label = {"roidb": entry}
    np.random.seed(seed)
    label.update(RPNTargets(max_size=max(H, W)).from_roidb(entry, 1.0, dev))
    label.update(PanopticLabels(dataset="cityscapes").from_roidb(entry, lmap, (H, W), 1.0, dev))
    data = {"data": TF.image(seed + 2, H, W).to(dev), "im_info": np.array([[H, W, 1.0]], np.float32)}
    return m, data, label


def _product_step(m, data, label, seed):
    m.keep_intermediates = True
    m.zero_grad(set_to_none=True)
    np.random.seed(seed)
    out = m(data, label)
    sum(out[k] for k in TF.LOSSES).backward()
    return out


def _oracle(m, depth, dconv, dev, dtype=torch.float64):
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    return TF.TrainOracle(sd, TF.trainable_names(m), depth=depth, dconv_from=dconv, dtype=dtype, device=dev)


def _compare(m, out, want, wgrads, prec, tag):
    named = dict(m.named_parameters())
    got = {k: (None if named[k].grad is None else named[k].grad) for k in wgrads}
    err = TF.grad_errors(got, wgrads)
    worst = max(err, key=err.get)
    plain = max((k for k in err if "offset" not in k), key=err.get)
    print("\n[%s %s] worst grad rel L2 outside the offset convs %.3e (%s)" % (tag, prec, err[plain], plain))
    lerr = {k: abs(float(out[k]) - want[k]) / max(abs(want[k]), 1e-3) for k in TF.LOSSES}
    lw = max(lerr, key=lerr.get)
    print("\n[%s %s] worst grad rel L2 %.3e (%s); worst loss rel %.3e (%s); accuracies %.4f/%.4f %.4f/%.4f"
          % (tag, prec, err[worst], worst, lerr[lw], lw, float(out["rcnn_accuracy"]), want["rcnn_accuracy"],
             float(out["panoptic_accuracy"]), want["panoptic_accuracy"]))
    bad = {k: e for k, e in err.items() if e > TF.grad_tol(k, prec)}
    assert not bad, bad
    assert lerr[lw] <= TF.LOSS_TOL[prec], (lw, lerr[lw])
    assert abs(float(out["rcnn_accuracy"]) - want["rcnn_accuracy"]) <= 0.02
    assert abs(float(out["panoptic_accuracy"]) - want["panoptic_accuracy"]) <= 0.02


@pytest.mark.parametrize("dconv", [100, 3])
@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_reduced_model_vs_oracle(dev, precision, prec, dconv):
    import upsnet_b200 as U
    depth = (2, 2, 2, 2)
    m, data, label = _setup(dev, dconv=dconv, depth=depth)
    U.set_precision(prec)
    buffers = {k: v.clone() for k, v in m.named_buffers()}
    frozen = {k: p.detach().clone() for k, p in m.named_parameters() if not p.requires_grad}
    out = _product_step(m, data, label, seed=5)
    assert set(k for k in out if k != "_intermediates") == set(TF.OUTPUTS)
    for k in TF.OUTPUTS:
        assert out[k].shape == (1,) and out[k].dtype == torch.float32 and out[k].is_cuda, k
    trainable = set(TF.trainable_names(m))
    for k, p in m.named_parameters():
        assert (p.grad is not None) == (k in trainable), k
    assert all(torch.equal(v, buffers[k]) for k, v in m.named_buffers())
    assert all(torch.equal(p, frozen[k]) for k, p in m.named_parameters() if k in frozen)
    want, wgrads = _oracle(m, depth, dconv, dev).step(data["data"], label, out["_intermediates"])
    _compare(m, out, want, wgrads, prec, "dconv=%d" % dconv)


def test_loss_parity_over_five_steps(dev, precision):
    import upsnet_b200 as U
    depth = (2, 2, 2, 2)
    m, data, label = _setup(dev, depth=depth, seed=3)
    U.set_precision("bf16x3")
    orc = _oracle(m, depth, 100, dev)
    groups = m.get_params_lr()
    names = {id(p): n for n, p in m.named_parameters()}
    ogroups = [dict({k: v for k, v in g.items() if k != "params"}, params=[orc.p[names[id(p)]] for p in g["params"]])
               for g in groups]
    opt = U.SGD(groups, lr=1, momentum=0.9, weight_decay=1e-4)
    oopt = OracleSGD(ogroups, lr=1, momentum=0.9, weight_decay=1e-4)
    first = None
    for step in range(5):
        out = _product_step(m, data, label, seed=10 + step)
        for p in orc.p.values():
            p.grad = None
        assert all(bool(torch.isfinite(out[k]).all()) for k in TF.OUTPUTS), step
        assert all(bool(torch.isfinite(p.grad).all()) for g in groups for p in g["params"]), step
        want, _ = orc.step(data["data"], label, out["_intermediates"])
        for k in TF.LOSSES:
            rel = abs(float(out[k]) - want[k]) / max(abs(want[k]), 1e-3)
            print("step %d %s %.6g %.6g rel %.2e" % (step, k, float(out[k]), want[k], rel))
            assert rel <= TF.LOSS_TOL["bf16x3"], (step, k, rel)
        first = first or {k: float(out[k]) for k in TF.LOSSES}
        opt.step(1e-7)          # the random-init heads have large gradients: keep the five steps in the smooth regime
        oopt.step(1e-7)
    # the updates reach the losses far beyond the tolerance, so the parity above is not parity of unchanged weights
    moved = [k for k in TF.LOSSES if abs(float(out[k]) - first[k]) > 20 * TF.LOSS_TOL["bf16x3"] * abs(first[k])]
    assert len(moved) >= 5, moved


@pytest.mark.parametrize("dconv", [100, 3])
def test_steps_match_a_model_built_from_the_updated_weights(dev, precision, dconv):
    """After every optimiser step, the model's training forward and backward equal those of a fresh model loaded with
    its state_dict: nothing packed, folded or cached from earlier weights survives a step (the offset convs included)."""
    import upsnet_b200 as U
    from upsnet_b200.model import UPSNetConfig, resnet_upsnet
    m, data, label = _setup(dev, dconv=dconv, seed=7)
    U.set_precision("bf16x3")
    opt = U.SGD(m.get_params_lr(), lr=1, momentum=0.9, weight_decay=1e-4)
    first = None
    for step in range(3):
        out = _product_step(m, data, label, seed=20 + step)
        assert all(bool(torch.isfinite(out[k]).all()) for k in TF.OUTPUTS), step
        if step:
            fresh = resnet_upsnet([2, 2, 2, 2], UPSNetConfig(backbone_with_dconv=dconv)).to(dev)
            fresh.load_state_dict(m.state_dict())
            want = _product_step(fresh, data, label, seed=20 + step)
            for k in TF.OUTPUTS:
                assert torch.equal(out[k], want[k]), (step, k, float(out[k]), float(want[k]))
            fg = {n: p.grad for n, p in fresh.named_parameters() if p.grad is not None}
            mg = {n: p.grad for n, p in m.named_parameters() if p.grad is not None}
            err = TF.grad_errors(mg, fg)
            assert max(err.values()) <= 1e-5, sorted(err.items(), key=lambda kv: -kv[1])[:3]
            moved = [k for k in TF.LOSSES if abs(float(out[k]) - first[k]) > 1e-3 * abs(first[k])]
            assert len(moved) >= 5, (step, moved)
        first = first or {k: float(out[k]) for k in TF.LOSSES}
        assert all(bool(torch.isfinite(p.grad).all()) for p in m.parameters() if p.grad is not None), step
        opt.step(1e-6)
        assert all(bool(torch.isfinite(p).all()) for p in m.parameters()), step


def test_inference_after_step_uses_updated_weights(dev, precision):
    import upsnet_b200 as U
    from upsnet_b200.model import UPSNetConfig, resnet_upsnet
    m, data, label = _setup(dev, seed=4)
    U.set_precision("bf16x3")
    with torch.no_grad():
        m(data)                     # a captured inference graph holding the old folded weights
    opt = U.SGD(m.get_params_lr(), lr=1, momentum=0.9, weight_decay=1e-4)
    _product_step(m, data, label, seed=1)
    opt.step(0.01)
    m.keep_intermediates = False
    got = m(data)
    fresh = resnet_upsnet([2, 2, 2, 2], UPSNetConfig()).to(dev)
    fresh.load_state_dict(m.state_dict())
    want = fresh(data)
    for k in ("cls_probs", "pred_boxes", "fcn_outputs", "panoptic_outputs"):
        assert torch.equal(got[k], want[k]), k


def test_full_size_step(dev, precision):
    import upsnet_b200 as U
    depth = (3, 4, 6, 3)
    m, data, label = _setup(dev, H=1024, W=2048, G=30, seed=6, depth=depth)
    U.set_precision("bf16x3")
    torch.cuda.reset_peak_memory_stats(dev)
    out = _product_step(m, data, label, seed=2)
    torch.cuda.synchronize(dev)
    peak = torch.cuda.max_memory_allocated(dev)
    print("\nfull-size R50 1024x2048 bf16x3 training step: peak memory %.2f GB" % (peak / 2 ** 30))
    for k in TF.OUTPUTS:
        assert torch.isfinite(out[k]).all(), k
    inter = out["_intermediates"]
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        torch.backends.cuda.matmul.allow_tf32 = False
        want = _oracle(m, depth, 100, dev, torch.float32).forward(data["data"], label, inter)
    for k in TF.LOSSES:
        rel = abs(float(out[k]) - float(want[k])) / max(abs(float(want[k])), 1e-3)
        print("full-size %s %.6g %.6g rel %.2e" % (k, float(out[k]), float(want[k]), rel))
        assert rel <= TF.LOSS_TOL["bf16x3"], (k, rel)
