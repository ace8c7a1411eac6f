"""Generates tests/golden/reference_panoptic_loss.npz by EXECUTING the reference's own SegTerm, MaskTerm
(operators/modules/unary_logits.py) and MaskMatching (operators/modules/mask_matching.py) under the lines of
models/resnet_upsnet.py that surround them in the training forward (build container only: /root/reference is not present
on the GPU box).  Run: python tests/golden/make_reference_panoptic_loss.py

models/resnet_upsnet.py itself cannot be imported (it pulls the un-buildable CUDA extensions), so `reference_head` below
replays its lines 156-179 and 250-257 on the reference modules and cites each line.  CPU, float32; the gradients are
autograd's.  Import shims as in make_reference_modules.py (easydict, the Cython modules, matplotlib); nothing inside the
executed functions is changed.

The cases come from tests/panoptic_loss_oracle.SMALL.  The file stores their inputs, the logits, the ground truth, loss,
accuracy and the gradients, with three economies that keep it small: mask_score is stored as its selected channels (the
others take no part); fcn_score, the one large random input, is stored as the sha256 of the array the seeded generator
builds (the tests rebuild it and check the digest before use); and of the logits only the instance and void channels
are stored, after checking here that the stuff channels are fcn_score's, bit for bit."""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_reference_modules as MRM  # noqa: E402  (puts /root/reference first on sys.path)
import panoptic_loss_oracle as PL  # noqa: E402


def reference_head(seg_term, mask_term, mask_matching, fcn_score, mask_score, gt_rois, cls_idx, seg_gt_4x, mask_gt, keep_inds,
                   enable_void, num_seg_classes, num_classes, mask_size):
    import torch
    import torch.nn as nn
    mask_score = mask_score.gather(1, cls_idx.view(-1, 1, 1, 1).expand(-1, -1, mask_size, mask_size))               # :156
    seg_logits, seg_inst_logits = seg_term(cls_idx, fcn_score, gt_rois)                                             # :159
    mask_logits = mask_term(mask_score, gt_rois, cls_idx, fcn_score)                                                # :160
    if enable_void:                                                                                                 # :162
        void_logits = torch.max(fcn_score[:, (num_seg_classes - num_classes + 1):, ...], dim=1, keepdim=True)[0] - \
            torch.max(seg_inst_logits, dim=1, keepdim=True)[0]                                                      # :163
        inst_logits = seg_inst_logits + mask_logits                                                                 # :164
        panoptic_logits = torch.cat([seg_logits, inst_logits, void_logits], dim=1)                                  # :165
    else:
        panoptic_logits = torch.cat([seg_logits, (seg_inst_logits + mask_logits)], dim=1)                           # :167
    with torch.no_grad():                                                                                           # :170
        if enable_void:
            panoptic_gt = mask_matching(seg_gt_4x, mask_gt, keep_inds=keep_inds)                                    # :172
        else:
            panoptic_gt = mask_matching(seg_gt_4x, mask_gt)                                                         # :174
    # calc_panoptic_acc, :250-257
    _, output_cls = torch.max(panoptic_logits.data, 1, keepdim=True)                                                # :251
    ignore = (panoptic_gt == 255).long().sum()                                                                      # :252
    correct = (output_cls.view(-1) == panoptic_gt.data.view(-1)).long().sum()                                       # :253
    total = (panoptic_gt.view(-1).shape[0]) - ignore                                                                # :254
    panoptic_acc = correct.float() / total.float()                                                                  # :256
    # self.panoptic_loss = nn.CrossEntropyLoss(ignore_index=255, reduce=False), :61
    panoptic_loss = nn.CrossEntropyLoss(ignore_index=255, reduction="none")(panoptic_logits, panoptic_gt)           # :178
    panoptic_loss = panoptic_loss.mean()                                                                            # :179
    return panoptic_logits, panoptic_gt, panoptic_loss, panoptic_acc, correct, ignore


def main():
    import torch
    MRM._install_shims()
    from upsnet.config.config import config
    MaskTerm, MaskMatching = MRM._reference_training_modules()
    from upsnet.operators.modules.unary_logits import SegTerm
    warnings.filterwarnings("ignore", message=".*upsample.*")
    out = {}
    for name, spec in PL.SMALL.items():
        c = PL.case(spec)
        S, nc, void = c["fcn"].shape[1], c["num_classes"], c["enable_void"]
        config.dataset.num_classes, config.dataset.num_seg_classes, config.network.mask_size = nc, S, 28
        fcn = torch.from_numpy(c["fcn"]).requires_grad_(True)
        msk = torch.from_numpy(c["mask_score"]).requires_grad_(True)
        logits, gt, loss, acc, correct, ignore = reference_head(
            SegTerm(S), MaskTerm(S), MaskMatching(S, void), fcn, msk, torch.from_numpy(c["rois"]), torch.from_numpy(c["cls"]),
            torch.from_numpy(c["seg_gt"]), torch.from_numpy(c["mask_gt"].astype(np.int64)), c["keep"], void, S, nc, 28)
        loss.backward()
        k = msk.shape[0]
        sel = msk.grad[torch.arange(k), torch.from_numpy(c["cls"])]
        rest = msk.grad.clone()
        rest[torch.arange(k), torch.from_numpy(c["cls"])] = 0
        assert not rest.any()
        p = name + "/"
        ns = S - nc + 1
        assert torch.equal(logits[:, :ns].detach(), fcn[:, :ns].detach())
        out.update({p + "fcn_sha256": np.str_(PL.digest(c["fcn"])), p + "mask_sel": PL.selected(c).numpy(), p + "rois": c["rois"], p + "cls": c["cls"],
                    p + "seg_gt": c["seg_gt"].astype(np.uint8), p + "mask_gt": c["mask_gt"],
                    p + "keep": c["keep"] if c["keep"] is not None else np.zeros(0, np.int64),
                    p + "logits_inst": logits[:, ns:].detach().numpy(), p + "gt": gt.numpy().astype(np.int64),
                    p + "loss": np.float32(loss.item()), p + "accuracy": np.float32(acc.item()),
                    p + "correct": np.int64(correct.item()), p + "ignored": np.int64(ignore.item()),
                    p + "d_fcn": fcn.grad.numpy(), p + "d_mask": sel.numpy()})
        print(name, "loss %.6f acc %.4f correct %d ignored %d channels %d" % (loss.item(), acc.item(), correct.item(),
                                                                              ignore.item(), logits.shape[1]))
    np.savez_compressed(os.path.join(HERE, "reference_panoptic_loss.npz"), **out)
    print("wrote reference_panoptic_loss.npz with", len(out), "arrays")


if __name__ == "__main__":
    main()
