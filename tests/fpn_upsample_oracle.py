"""The literal model and the training-step oracle with the reference's bilinear FPN (network.fpn_upsample_method =
'bilinear') -- TEST INFRASTRUCTURE ONLY.

models/fpn.py:27-35 builds fpn_upsample as F.interpolate(x, scale_factor=2, mode=upsample_method, align_corners=False
if bilinear) and applies it three times on the top-down path (:88-93).  BilinearLiteralUPSNet restates FPN.forward
(fpn.py:78-104) with that up-sampling materialised; every other layer, and the nearest FPN, stay those of
oracle/literal_model.LiteralUPSNet.  BilinearTrainOracle is train_forward_oracle.TrainOracle on that graph: its fpn
(the planted P6 fault) and gap (fpn_gap with its gradient) run around this FPN."""
import torch.nn.functional as F

import train_forward_oracle as TF
from oracle.literal_model import LiteralUPSNet


class BilinearLiteralUPSNet(LiteralUPSNet):
    def fpn(self, res2, res3, res4, res5):
        up = lambda t: F.interpolate(t, scale_factor=2, mode="bilinear", align_corners=False)     # noqa: E731
        p5_1x1 = self.fpn_conv(res5, "fpn.fpn_p5_1x1")
        if self.with_gap:
            p5_1x1 = p5_1x1 + self.gap(res5)               # fpn.py:84-88: the context vector before the up-sampling
        p4_plus = up(p5_1x1) + self.fpn_conv(res4, "fpn.fpn_p4_1x1")
        p3_plus = up(p4_plus) + self.fpn_conv(res3, "fpn.fpn_p3_1x1")
        p2_plus = up(p3_plus) + self.fpn_conv(res2, "fpn.fpn_p2_1x1")
        p2 = self.fpn_conv(p2_plus, "fpn.fpn_p2", 1)
        p3 = self.fpn_conv(p3_plus, "fpn.fpn_p3", 1)
        p4 = self.fpn_conv(p4_plus, "fpn.fpn_p4", 1)
        p5 = self.fpn_conv(p5_1x1, "fpn.fpn_p5", 1)
        p6 = F.max_pool2d(p5, 1, 2)
        return p2, p3, p4, p5, p6


class BilinearTrainOracle(TF.TrainOracle, BilinearLiteralUPSNet):
    """TrainOracle.fpn calls super().fpn, which resolves to BilinearLiteralUPSNet.fpn."""
