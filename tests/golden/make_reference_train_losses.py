"""Generates tests/golden/reference_train_losses.npz by EXECUTING the reference's own RPNLoss (models/rpn.py:60-92) and
MaskRCNNLoss (models/rcnn.py:159-197), and the semantic-loss lines of the training forward (build container only:
/root/reference is not present on the GPU box).  Run: python tests/golden/make_reference_train_losses.py

models/rpn.py and models/rcnn.py are loaded by file path after make_reference_modules' import shims, with a stub for the
un-buildable roi_align extension that rcnn.py's imports reach (nothing the losses run touches it).  The semantic loss
comes from models/fcn.py:101 and models/resnet_upsnet.py:79,131, which cannot be imported (the model pulls every CUDA
extension), so `reference_fcn_loss` replays those lines and cites each.  CPU, float32; the gradients are autograd's.

The cases come from tests/train_loss_oracle (SEM_SMALL, RPN_SMALL, MRCNN_SMALL).  To stay small the file stores the
seeded generators' inputs as their sha256 (the tests rebuild them and check the digest before use), and the outputs:
losses, counts, accuracy and gradients."""
import importlib.util
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_reference_modules as MRM  # noqa: E402  (puts /root/reference first on sys.path)
import train_loss_oracle as TL  # noqa: E402

REF = "/root/reference/upsnet/models"


def _load(name):
    spec = importlib.util.spec_from_file_location("ref_" + name, os.path.join(REF, name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def reference_modules():
    MRM._install_shims()
    ext = types.ModuleType("upsnet.operators._ext.roi_align")
    ext.roi_align_cuda = None
    sys.modules.setdefault("upsnet.operators._ext", types.ModuleType("upsnet.operators._ext"))
    sys.modules["upsnet.operators._ext.roi_align"] = ext
    return _load("rpn").RPNLoss, _load("rcnn").MaskRCNNLoss


def reference_fcn_loss(fcn_score, seg_gt):
    import torch.nn as nn
    import torch.nn.functional as F
    output = F.interpolate(fcn_score, None, 4, mode='bilinear', align_corners=False)    # models/fcn.py:101
    fcn_loss = nn.CrossEntropyLoss(ignore_index=255)                                      # models/resnet_upsnet.py:79
    return fcn_loss(output, seg_gt)                                                       # models/resnet_upsnet.py:131


def main():
    import torch
    RPNLoss, MaskRCNNLoss = reference_modules()
    out = {}
    for name, spec in TL.SEM_SMALL.items():
        seed, S, h, w, pad, ign, _ = spec
        c = TL.semantic_case(seed, S, h, w, pad, ign)
        x = torch.from_numpy(c["fcn"]).requires_grad_(True)
        loss = reference_fcn_loss(x, torch.from_numpy(c["seg_gt"]).long())
        loss.backward()
        p = "sem/%s/" % name
        out.update({p + "inputs_sha256": np.str_(TL.digest(c["fcn"]) + TL.digest(c["seg_gt"])),
                    p + "loss": np.float32(loss.item()), p + "n": np.int64((c["seg_gt"] != 255).sum()),
                    p + "d_fcn": x.grad.numpy()})
        print("semantic", name, "loss %.6f" % loss.item())
    for name, spec in TL.RPN_SMALL.items():
        seed, ih, iw, field = spec
        c = TL.rpn_case(seed, ih, iw, field)
        xs = [torch.from_numpy(a).requires_grad_(True) for a in c["scores"]]
        ps = [torch.from_numpy(a).requires_grad_(True) for a in c["preds"]]
        lab = {k: torch.from_numpy(v) for k, v in c["label"].items()}
        cls_loss, bbox_loss = RPNLoss(256)(xs, ps, lab)
        (cls_loss + bbox_loss).backward()
        p = "rpn/%s/" % name
        out.update({p + "inputs_sha256": np.str_("".join(TL.digest(a) for a in c["scores"] + c["preds"]) +
                                                  "".join(TL.digest(c["label"][k]) for k in sorted(c["label"]))),
                    p + "cls_loss": np.float32(cls_loss.item()), p + "bbox_loss": np.float32(bbox_loss.item())})
        for s, x, q in zip(TL.STRIDES, xs, ps):
            out[p + "d_score%d" % s] = x.grad.numpy()
            out[p + "d_pred%d" % s] = q.grad.numpy()
        print("rpn", name, "cls %.6f bbox %.6f" % (cls_loss.item(), bbox_loss.item()))
    from upsnet.config.config import config
    for name, spec in TL.MRCNN_SMALL.items():
        seed, R, K, n, M, ign, none = spec
        c = TL.mask_rcnn_case(seed, R, K, n, M, ign, none)
        config.network.mask_size = M
        t = {k: torch.from_numpy(c[k]) for k in TL.NAMES}
        for k in ("cls_score", "bbox_pred", "mask_score"):
            t[k].requires_grad_(True)
        cls_loss, bbox_loss, mask_loss, acc = MaskRCNNLoss(512)(*(t[k] for k in TL.NAMES))
        (cls_loss + bbox_loss + mask_loss).backward()
        p = "mrcnn/%s/" % name
        out.update({p + "inputs_sha256": np.str_("".join(TL.digest(c[k]) for k in TL.NAMES)),
                    p + "cls_loss": np.float32(cls_loss.item()), p + "bbox_loss": np.float32(bbox_loss.item()),
                    p + "mask_loss": np.float32(mask_loss.item()), p + "accuracy": np.float32(acc.item()),
                    p + "d_cls": t["cls_score"].grad.numpy(), p + "d_bbox": t["bbox_pred"].grad.numpy(),
                    p + "d_mask": t["mask_score"].grad.numpy()})
        print("mask_rcnn", name, "cls %.6f bbox %.6f mask %.6f acc %.4f" % (cls_loss.item(), bbox_loss.item(),
                                                                          mask_loss.item(), acc.item()))
    np.savez_compressed(os.path.join(HERE, "reference_train_losses.npz"), **out)
    print("wrote reference_train_losses.npz with", len(out), "arrays")


if __name__ == "__main__":
    main()
