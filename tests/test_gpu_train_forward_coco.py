"""The training forward of the COCO configurations on the device (UPSNetConfig.coco_r50: fpn_with_gap,
fcn_with_roi_loss, fcn_num_layers 3, 81 / 133 classes) against the float64 oracle of tests/train_forward_oracle.py,
with the criteria of tests/test_gpu_train_forward.py (train_forward_oracle.LOSS_TOL / grad_tol).

The synthetic model calibrates the FPN laterals to RMS 1 but leaves fpn_gap at the reference's nn.Linear
initialisation, which on a random-init res5 gives a context vector of RMS ~60: every FPN level is then a near-constant
offset, the RCNN logits saturate and a comparison with float64 measures that conditioning rather than the step.
_calibrate_gap scales fpn_gap so that its context vector has RMS 1 on the test image, as the laterals have."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import train_forward_oracle as TF  # noqa: E402

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


def _calibrate_gap(m, x):
    with torch.no_grad():
        r5 = m.resnet_backbone.forward_train(x, "bf16x3")[3]
        g = TF.gap_vector(r5, m.fpn.fpn_gap.weight, m.fpn.fpn_gap.bias)
        s = 1.0 / float(g.pow(2).mean().sqrt())
        m.fpn.fpn_gap.weight.mul_(s)
        m.fpn.fpn_gap.bias.mul_(s)


def _config(dconv):
    from upsnet_b200.model import UPSNetConfig
    cfg = UPSNetConfig.coco_r50()
    cfg.backbone_with_dconv = dconv
    return cfg


def _setup(dev, dconv=100, H=256, W=512, G=8, seed=0, depth=(2, 2, 2, 2)):
    from upsnet_b200.synthetic import synthetic_model
    from upsnet_b200.training import PanopticLabels, RPNTargets
    m = synthetic_model(_config(dconv), depth=depth, seed=seed, device=dev)
    entry, lmap = TF.synthetic_entry(seed + 1, H, W, G, num_classes=81)
    label = {"roidb": entry}
    np.random.seed(seed)
    label.update(RPNTargets(max_size=max(H, W)).from_roidb(entry, 1.0, dev))
    label.update(PanopticLabels(dataset="coco", with_roi=True).from_roidb(entry, lmap, (H, W), 1.0, dev))
    data = {"data": TF.image(seed + 2, H, W).to(dev), "im_info": np.array([[H, W, 1.0]], np.float32)}
    _calibrate_gap(m, data["data"])
    return m, data, label


def _product_step(m, data, label, seed):
    m.keep_intermediates = True
    m.zero_grad(set_to_none=True)
    np.random.seed(seed)
    out = m(data, label)
    sum(out[k] for k in TF.COCO_LOSSES).backward()
    return out


def _oracle(m, depth, dconv, dev, dtype=torch.float64, **kw):
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    return TF.TrainOracle(sd, TF.trainable_names(m), depth=depth, num_classes=81, num_seg_classes=133, dconv_from=dconv,
                          fcn_layers=3, with_gap=True, fcn_with_roi_loss=True, dtype=dtype, device=dev, **kw)


def _errors(m, out, want, wgrads):
    named = dict(m.named_parameters())
    err = TF.grad_errors({k: named[k].grad for k in wgrads}, wgrads)
    lerr = {k: abs(float(out[k]) - want[k]) / max(abs(want[k]), 1e-3) for k in TF.COCO_LOSSES}
    return err, lerr


def _rejected(err, lerr, prec):
    return any(e > TF.grad_tol(k, prec) for k, e in err.items()) or any(e > TF.LOSS_TOL[prec] for e in lerr.values())


@pytest.mark.parametrize("dconv", [100, 3])
@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_reduced_coco_model_vs_oracle(dev, precision, prec, dconv):
    import upsnet_b200 as U
    depth = (2, 2, 2, 2)
    m, data, label = _setup(dev, dconv=dconv, depth=depth)
    U.set_precision(prec)
    out = _product_step(m, data, label, seed=5)
    assert set(k for k in out if k != "_intermediates") == set(TF.OUTPUTS) | {"fcn_roi_loss"}
    for k in TF.OUTPUTS:
        assert out[k].shape == (1,) and out[k].dtype == torch.float32 and out[k].is_cuda, k
    r = out["fcn_roi_loss"]
    assert r.shape == () and r.dtype == torch.float32 and r.is_cuda and bool(torch.isfinite(r))
    inter = out["_intermediates"]
    assert inter["fcn_rois"].shape[0] == label["seg_roi_gt"].shape[0] >= inter["gt_rois"].shape[0]
    trainable = set(TF.trainable_names(m))
    assert {"fpn.fpn_gap.weight", "fpn.fpn_gap.bias"} <= trainable
    for k, p in m.named_parameters():
        assert (p.grad is not None) == (k in trainable), k
    assert float(m.fpn.fpn_gap.weight.grad.abs().sum()) > 0
    want, wgrads = _oracle(m, depth, dconv, dev).step(data["data"], label, inter)
    err, lerr = _errors(m, out, want, wgrads)
    worst, lw = max(err, key=err.get), max(lerr, key=lerr.get)
    print("\n[coco dconv=%d %s] worst grad rel L2 %.3e (%s); fpn_gap %.3e; worst loss rel %.3e (%s); fcn_roi_loss %.3e"
          % (dconv, prec, err[worst], worst, err["fpn.fpn_gap.weight"], lerr[lw], lw, lerr["fcn_roi_loss"]))
    bad = {k: e for k, e in err.items() if e > TF.grad_tol(k, prec)}
    assert not bad, bad
    assert lerr[lw] <= TF.LOSS_TOL[prec], (lw, lerr[lw])
    # the planted faults: the same criteria reject an oracle without the gap's gradient, or whose ROI loss takes the
    # kept boxes only
    if prec == "bf16x3" and dconv == 100:
        for fault in TF.COCO_FAULTS:
            fw, fg = _oracle(m, depth, dconv, dev, fault=fault).step(data["data"], label, inter)
            assert _rejected(*_errors(m, out, fw, fg), prec), fault


@pytest.mark.parametrize("dconv", [100, 3])
def test_steps_match_a_model_built_from_the_updated_weights(dev, precision, dconv):
    """Three SGD steps: after each, the training forward equals bit for bit that of a fresh model loaded with the
    state_dict, fpn_gap and the ROI loss included."""
    import upsnet_b200 as U
    from upsnet_b200.model import resnet_upsnet
    m, data, label = _setup(dev, dconv=dconv, seed=7)
    U.set_precision("bf16x3")
    opt = U.SGD(m.get_params_lr(), lr=1, momentum=0.9, weight_decay=1e-4)
    outs = TF.OUTPUTS + ("fcn_roi_loss",)
    gap0 = m.fpn.fpn_gap.weight.detach().clone()
    for step in range(3):
        out = _product_step(m, data, label, seed=20 + step)
        assert all(bool(torch.isfinite(out[k]).all()) for k in outs), step
        if step:
            fresh = resnet_upsnet([2, 2, 2, 2], _config(dconv)).to(dev)
            fresh.load_state_dict(m.state_dict())
            want = _product_step(fresh, data, label, seed=20 + step)
            for k in outs:
                assert torch.equal(out[k], want[k]), (step, k, float(out[k]), float(want[k]))
            fg = {n: p.grad for n, p in fresh.named_parameters() if p.grad is not None}
            mg = {n: p.grad for n, p in m.named_parameters() if p.grad is not None}
            err = TF.grad_errors(mg, fg)
            assert max(err.values()) <= 1e-5, sorted(err.items(), key=lambda kv: -kv[1])[:3]
        opt.step(1e-6)
    assert not torch.equal(m.fpn.fpn_gap.weight, gap0)


def test_full_size_coco_step(dev, precision):
    import upsnet_b200 as U
    depth = (3, 4, 6, 3)
    m, data, label = _setup(dev, H=800, W=1344, G=30, seed=6, depth=depth)
    U.set_precision("bf16x3")
    torch.cuda.reset_peak_memory_stats(dev)
    out = _product_step(m, data, label, seed=2)
    torch.cuda.synchronize(dev)
    peak = torch.cuda.max_memory_allocated(dev)
    print("\nfull-size R50 COCO 800x1344 bf16x3 training step: peak memory %.2f GB" % (peak / 2 ** 30))
    for k in TF.OUTPUTS + ("fcn_roi_loss",):
        assert torch.isfinite(out[k]).all(), k
    inter = out["_intermediates"]
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        torch.backends.cuda.matmul.allow_tf32 = False
        want = _oracle(m, depth, 100, dev, torch.float32).forward(data["data"], label, inter)
    for k in TF.COCO_LOSSES:
        rel = abs(float(out[k]) - float(want[k])) / max(abs(float(want[k])), 1e-3)
        print("full-size %s %.6g %.6g rel %.2e" % (k, float(out[k]), float(want[k]), rel))
        assert rel <= TF.LOSS_TOL["bf16x3"], (k, rel)
