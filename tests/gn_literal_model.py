"""The group_norm heads of the reference (network.{fpn,rcnn,fcn}_with_norm = 'group_norm') restated in plain torch, on
top of the literal model (oracle/literal_model.py) and the training-step oracle (tests/train_forward_oracle.py).

The mixin overrides the FPN, the FCN sub-network, RCNN fc6 and the mask convs when the state_dict carries their
GroupNorm parameters (reference key names: fpn.fpn_p5_1x1.{0,1}, fcn_head.fcn_subnet.conv.i.{0,1}, rcnn.fc6.{0,2},
mask_branch.mask_convN.{0,1}), and defers to the plain graph otherwise, so a 'none' state_dict runs today's graph.
Reference lines restated (paths relative to /root/reference/upsnet/models/):
  fpn.py:43-58 and :78-104 (conv without bias -> GroupNorm(32), the context vector added after the GN of fpn_p5_1x1)
  fcn.py:41-52 (DeformConvWithOffset -> GroupNorm(32) -> ReLU)
  rcnn.py:50-56 (mask convs without bias -> GroupNorm(32) -> ReLU), :102 (fc6: Linear -> view [R,C,1,1] -> GN -> ReLU)
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle.literal_model import LiteralUPSNet  # noqa: E402
import train_forward_oracle as TF  # noqa: E402


def fixture_values(seed, shape, scale=1.0, offset=0.0):
    """Deterministic float32 values, uniform in offset + scale * [-1/2, 1/2), defined by this code alone (splitmix64
    keys of upsnet_b200.training.draw_keys, top 24 bits): the FPN / RPN inputs and parameters of
    tests/golden/make_reference_group_norm.py, made again by the test instead of being stored in the fixture."""
    from upsnet_b200.training import draw_keys
    n = int(np.prod(shape))
    u = (draw_keys(seed, n) >> np.uint64(40)).astype(np.float64) / 2.0 ** 24
    return torch.from_numpy(((u - 0.5) * scale + offset).astype(np.float32).reshape(shape))


def fixture_fpn_params(shapes):
    """{name: tensor} for the (name, shape) list of the reference FPN / RPN parameters, in order: GroupNorm weights
    around 1, other biases and GN biases around 0 (scale 0.4), weights at scale 0.1."""
    out = {}
    for i, (name, shape) in enumerate(shapes):
        gn_w = name.endswith(".1.weight")
        out[name] = fixture_values(1000 + i, shape, 0.4 if len(shape) == 1 else 0.1, 1.0 if gn_w else 0.0)
    return out


class GroupNormMixin:
    def gn(self, x, name):
        return F.group_norm(x, 32, self.p[name + ".weight"], self.p[name + ".bias"], 1e-5)

    def fpn(self, res2, res3, res4, res5):
        if "fpn.fpn_p5_1x1.1.weight" not in self.p:
            return super().fpn(res2, res3, res4, res5)
        up = lambda t: F.interpolate(t, scale_factor=2, mode="nearest")     # noqa: E731
        c = lambda x, n, pad=0: self.gn(F.conv2d(x, self.p[n + ".0.weight"], None, 1, pad), n + ".1")   # noqa: E731
        p5_1x1 = c(res5, "fpn.fpn_p5_1x1")
        if self.with_gap:
            p5_1x1 = p5_1x1 + self.gap(res5)
        p4_plus = up(p5_1x1) + c(res4, "fpn.fpn_p4_1x1")
        p3_plus = up(p4_plus) + c(res3, "fpn.fpn_p3_1x1")
        p2_plus = up(p3_plus) + c(res2, "fpn.fpn_p2_1x1")
        p2 = c(p2_plus, "fpn.fpn_p2", 1)
        p3 = c(p3_plus, "fpn.fpn_p3", 1)
        p4 = c(p4_plus, "fpn.fpn_p4", 1)
        p5 = c(p5_1x1, "fpn.fpn_p5", 1)
        return p2, p3, p4, p5, F.max_pool2d(p5, 1, 2)

    def fcn_level(self, x, level):
        if "fcn_head.fcn_subnet.conv.0.1.weight" not in self.p:
            return super().fcn_level(x, level)
        for i in range(self.fcn_layers):
            p = "fcn_head.fcn_subnet.conv.%d" % i
            offset = self.conv(x, p + ".0.conv_offset", 1, 1, 1)
            x = F.relu(self.gn(self.dcn(x, offset, p + ".0.conv"), p + ".1"))
        return x

    def rcnn(self, feats, rois):
        if "rcnn.fc6.2.weight" not in self.p:
            return super().rcnn(feats, rois)
        x = self.fpn_roi_align(feats, rois, 7).flatten(1)
        fc6 = F.linear(x, self.p["rcnn.fc6.0.weight"], self.p["rcnn.fc6.0.bias"])
        fc6 = F.relu(self.gn(fc6.view(fc6.shape[0], -1, 1, 1), "rcnn.fc6.2").flatten(1))
        fc7 = F.relu(F.linear(fc6, self.p["rcnn.fc7.0.weight"], self.p["rcnn.fc7.0.bias"]))
        return {"cls_score": F.linear(fc7, self.p["rcnn.cls_score.weight"], self.p["rcnn.cls_score.bias"]),
                "bbox_pred": F.linear(fc7, self.p["rcnn.bbox_pred.weight"], self.p["rcnn.bbox_pred.bias"]), "fc_feat": fc7}

    def mask_branch(self, feats, rois):
        if "mask_branch.mask_conv1.1.weight" not in self.p:
            return super().mask_branch(feats, rois)
        x = self.fpn_roi_align(feats, rois, 14)
        for i in range(1, 5):
            x = F.relu(self.gn(self.conv(x, "mask_branch.mask_conv%d.0" % i, 1, 1), "mask_branch.mask_conv%d.1" % i))
        x = F.relu(F.conv_transpose2d(x, self.p["mask_branch.mask_deconv1.0.weight"],
                                      self.p["mask_branch.mask_deconv1.0.bias"], 2))
        return self.conv(x, "mask_branch.mask_score")


class LiteralGNUPSNet(GroupNormMixin, LiteralUPSNet):
    pass


class GNTrainOracle(GroupNormMixin, TF.TrainOracle):
    pass
