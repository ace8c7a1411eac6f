"""The float64 training-step oracle of the COCO configurations: train_forward_oracle.TrainOracle plus FPN's global
context branch (models/fpn.py:84-86: fpn_p5_1x1 + fpn_gap(GAP(res5)), broadcast) and the semantic head's ROI loss
(models/fcn.py:102-106, models/resnet_upsnet.py:132-134), restated literally: RoIAlign of the 512-channel concat, the
score conv, the cross-entropy with ignore_index 255 averaged over every cell.  The ROI loss takes the product's
'fcn_rois' (every ground-truth box, before the keep draw).

Planted faults (COCO_FAULTS): 'gap_detached' (no gradient through fpn_gap), 'rois_after_keep' (the ROI loss on the kept
boxes and their seg_roi_gt rows only)."""
import torch
import torch.nn.functional as F

import fcn_roi_loss_oracle as FO
import train_forward_oracle as TF

COCO_FAULTS = ("gap_detached", "rois_after_keep")
LOSSES = TF.LOSSES + ("fcn_roi_loss",)


def gap_vector(res5, weight, bias, detached=False):
    """models/fpn.py:85: fpn_gap(adaptive_avg_pool2d(res5, 1)) as [1, C, 1, 1]."""
    if detached:
        res5, weight, bias = res5.detach(), weight.detach(), bias.detach()
    return F.linear(F.adaptive_avg_pool2d(res5, (1, 1)).flatten(1), weight, bias).view(1, -1, 1, 1)


def roi_loss(feat, weight, bias, rois, seg, keep=None):
    """The reference's fcn_roi_loss from the 512-channel concat feat [1,512,h,w]; with keep, the faulty variant that
    takes only the kept boxes (and their rows)."""
    if keep is not None:
        keep = torch.as_tensor(keep, device=rois.device).long()
        rois, seg = rois[keep], seg[keep]
    f = feat[0]
    By, Bx, _ = FO.roi_align_weights(rois, f.shape[1], f.shape[2], seg.shape[1])
    rf = torch.einsum("rmy,cyx,rnx->rcmn", By.to(f.dtype), f, Bx.to(f.dtype))
    return FO.ce_mean(F.conv2d(rf, weight, bias), seg.long())


class CocoTrainOracle(TF.TrainOracle):
    def __init__(self, *args, coco_fault=None, **kw):
        assert coco_fault is None or coco_fault in COCO_FAULTS
        super().__init__(*args, **kw)
        self.coco_fault = coco_fault

    def conv(self, x, name, stride=1, padding=0, dilation=1):
        if name == "fcn_head.score":
            self._feat = x                            # the 512-channel concat, for the ROI loss
        y = super().conv(x, name, stride, padding, dilation)
        if name == "fpn.fpn_p5_1x1":
            y = y + gap_vector(x, self.p["fpn.fpn_gap.weight"], self.p["fpn.fpn_gap.bias"],
                               self.coco_fault == "gap_detached")
        return y

    def forward(self, image, label, inter):
        out = super().forward(image, label, inter)
        keep = inter["keep_inds"] if self.coco_fault == "rois_after_keep" else None
        out["fcn_roi_loss"] = roi_loss(self._feat, self.p["fcn_head.score.weight"], self.p["fcn_head.score.bias"],
                                       inter["fcn_rois"].to(self.device), label["seg_roi_gt"].to(self.device), keep)
        return out

    def step(self, image, label, inter):
        out = self.forward(image, label, inter)
        sum(out[k] for k in LOSSES).backward()
        return {k: float(v.detach()) if torch.is_tensor(v) else float(v) for k, v in out.items()}, self.grads()
