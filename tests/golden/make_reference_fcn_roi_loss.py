"""Generates tests/golden/reference_fcn_roi_loss.npz by EXECUTING the reference's semantic-head ROI loss (build container
only: /root/reference is not present on the GPU box).  Run: python tests/golden/make_reference_fcn_roi_loss.py

* FCNHead.forward is taken from upsnet/models/fcn.py by its AST and run unmodified on an object whose fcn_subnet is the
  identity (the cases give the four subnet outputs), whose score is an nn.Conv2d(512, S, 1) with the case's weights,
  and whose roipool is torchvision's roi_align(output_size 28, spatial_scale 1/4, sampling_ratio 2, aligned=False), the
  binding SURVEY section 8c verified against the reference's RoIAlign.
* The loss lines upsnet/models/resnet_upsnet.py:132-134 are run unmodified, with self.fcn_roi_loss =
  nn.CrossEntropyLoss(ignore_index=255, reduce=False) as resnet_upsnet.__init__ builds it.

Written per case of tests/fcn_roi_loss_oracle.CASES, on CPU float32 with one thread: the digest of the seeded inputs,
the loss, and the gradients of the score conv's weight and bias.  Fixed member timestamps: a second run gives the same
bytes."""
import ast
import os
import sys
import textwrap
import types
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import fcn_roi_loss_oracle as O  # noqa: E402
from make_reference_sgd import save_npz  # noqa: E402

REF = "/root/reference/upsnet/models"


def reference_fcn_forward(ns):
    path = os.path.join(REF, "fcn.py")
    tree = ast.parse(open(path).read(), path)
    cls = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "FCNHead"][0]
    fn = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "forward"][0]
    exec(compile(ast.Module(body=[fn], type_ignores=[]), path, "exec"), ns)
    return ns["forward"]


def reference_loss_lines():
    path = os.path.join(REF, "resnet_upsnet.py")
    lines = open(path).read().split("\n")[131:134]           # lines 132-134
    assert "fcn_with_roi_loss" in lines[0] and "fcn_roi_loss.mean()" in lines[2], lines
    return compile(textwrap.dedent("\n".join(lines)), path, "exec")


def main():
    import torch
    import torch.nn as nn
    import torch.nn.functional as F
    from torchvision.ops import roi_align
    torch.set_num_threads(1)
    warnings.filterwarnings("ignore", message=".*reduce.*")
    forward = reference_fcn_forward({"torch": torch, "nn": nn, "F": F})
    loss_code = reference_loss_lines()
    config = types.SimpleNamespace(train=types.SimpleNamespace(fcn_with_roi_loss=True))
    out = {}
    for name in O.CASES:
        c = O.case(name)
        S = c["weight"].shape[0]
        head = types.SimpleNamespace(fcn_subnet=lambda x: x, upsample_rate=4, score=nn.Conv2d(512, S, 1),
                                     roipool=lambda feat, roi: roi_align(feat, roi, (O.M, O.M), O.SCALE, O.SR,
                                                                         aligned=False))
        with torch.no_grad():
            head.score.weight.copy_(c["weight"])
            head.score.bias.copy_(c["bias"])
        fcn_output = forward(head, *c["levels"], c["rois"])
        ns = {"self": types.SimpleNamespace(fcn_roi_loss=nn.CrossEntropyLoss(ignore_index=255, reduce=False)),
              "fcn_output": fcn_output, "label": {"seg_roi_gt": c["seg"]}, "config": config}
        exec(loss_code, ns)
        loss = ns["fcn_roi_loss"]
        loss.backward()
        p = "case/%s/" % name
        out[p + "inputs_sha256"] = np.str_(O.inputs_digest(c))
        out[p + "loss"] = np.float32(loss.item())
        out[p + "d_weight"] = head.score.weight.grad.numpy().reshape(S, 512).copy()
        out[p + "d_bias"] = head.score.bias.grad.numpy().copy()
        print(name, "loss %.7f" % loss.item())
    save_npz(os.path.join(HERE, "reference_fcn_roi_loss.npz"), out)


if __name__ == "__main__":
    main()
