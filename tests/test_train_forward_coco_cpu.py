"""The COCO pieces of the training oracle (tests/train_forward_oracle.py) on CPU: its ROI loss reproduces the
reference fixture (tests/golden/reference_fcn_roi_loss.npz), and the criteria of the GPU comparison reject its two
planted faults, the ROI loss on the boxes kept by the panoptic draw and a context vector detached from fpn_gap."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import fcn_roi_loss_oracle as FO  # noqa: E402
import train_forward_oracle as TF  # noqa: E402

Z = np.load(os.path.join(HERE, "golden", "reference_fcn_roi_loss.npz"))


def test_roi_loss_matches_the_reference_and_rejects_the_kept_boxes():
    name = "s133_r90"
    c = FO.case(name)
    assert FO.inputs_digest(c) == str(Z["case/%s/inputs_sha256" % name])
    feat = FO.feat_of(c["levels"])
    R = c["rois"].shape[0]
    keep = np.random.default_rng(3).choice(R, max(int(R * 0.7), 1), replace=False)   # resnet_upsnet.py:149's draw
    out = {}
    for k in (None, keep):
        w, b = c["weight"].double().requires_grad_(True), c["bias"].double().requires_grad_(True)
        loss = TF.roi_loss(feat, w, b, c["rois"], c["seg"], keep=k)
        loss.backward()
        out[k is None] = (float(loss), {"fcn_head.score.weight": w.grad, "fcn_head.score.bias": b.grad})
    want = float(Z["case/%s/loss" % name])
    assert abs(out[True][0] - want) <= 1e-5 * abs(want)
    err = TF.grad_errors(out[False][1], out[True][1])
    assert all(e > TF.grad_tol(k, "bf16x3") for k, e in err.items()), err

def test_detached_gap_is_rejected():
    g = torch.Generator().manual_seed(0)
    res5 = torch.rand(1, 2048, 4, 6, generator=g, dtype=torch.float64).requires_grad_(True)
    grads = {}
    for detached in (False, True):
        w = (torch.randn(256, 2048, generator=g, dtype=torch.float64) * 0.02).requires_grad_(True)
        bias = torch.randn(256, generator=g, dtype=torch.float64).requires_grad_(True)
        v = TF.gap_vector(res5, w, bias, detached)
        assert v.shape == (1, 256, 1, 1)
        if not detached:
            ref = torch.nn.functional.linear(res5.mean((2, 3)), w, bias)
            assert torch.allclose(v.flatten(1), ref, rtol=1e-12, atol=0)
            (v * torch.arange(256, dtype=torch.float64).view(1, -1, 1, 1)).sum().backward()
        grads[detached] = {"fpn.fpn_gap.weight": w.grad, "fpn.fpn_gap.bias": bias.grad}
    err = TF.grad_errors(grads[True], grads[False])
    assert all(e > TF.grad_tol(k, "bf16") for k, e in err.items())
