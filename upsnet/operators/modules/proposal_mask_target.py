"""reference path: upsnet/operators/modules/proposal_mask_target.py:27-62"""
from torch.nn import Module

from upsnet_b200.training import ProposalTargets


class ProposalMaskTarget(Module):
    """The reference's module on the device: forward(rois, roidb, im_info) returns the same nine tensors (rois, labels,
    bbox_targets, bbox_inside_weights, bbox_outside_weights, mask_rois, mask_int32, roi_has_mask, nongt_inds) with one
    synchronisation instead of the host round trip.  num_classes and fg_fraction come from the arguments; batch_rois,
    the thresholds, the box weights and the mask size from the reference's `config` when it is importable."""

    def __init__(self, num_classes, batch_images, batch_rois, fg_fraction, mask_size, binary_thresh):
        super(ProposalMaskTarget, self).__init__()
        self.num_classes, self.batch_images, self.batch_rois = num_classes, batch_images, batch_rois
        self.fg_fraction, self.mask_size, self.binary_thresh = fg_fraction, mask_size, binary_thresh
        kw = {}
        try:
            from upsnet.config.config import config
            tr, net = config.train, config.network
            kw = dict(fg_thresh=tr.fg_thresh, bg_thresh_hi=tr.bg_thresh_hi, bg_thresh_lo=tr.bg_thresh_lo,
                      bbox_reg_weights=net.bbox_reg_weights, cls_agnostic_bbox_reg=net.cls_agnostic_bbox_reg)
        except (ImportError, AttributeError):
            pass
        self.targets = ProposalTargets(num_classes=num_classes, batch_rois=batch_rois, fg_fraction=fg_fraction,
                                       mask_size=mask_size, **kw)

    def forward(self, rois, roidb, im_info):
        assert self.batch_rois == -1 or self.batch_rois % self.batch_images == 0, \
            'batchimages {} must devide batch_rois {}'.format(self.batch_images, self.batch_rois)
        return self.targets.from_roidb(rois, roidb, im_info)
