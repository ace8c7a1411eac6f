"""Literal restatement of the reference's model graph in plain torch -- TEST INFRASTRUCTURE ONLY.

An INDEPENDENT whole-model oracle (VERDICT r1 "missing" item 4): unlike oracle/cpu_model.py, which runs the product's own
`upsnet_b200.model` graph with CPU ops plugged in, nothing here shares code with the product.  The graph is written the
way the reference writes it -- un-folded eval-mode BatchNorm, ConvTranspose2d, up-sample -> concat -> score, separate
cls / bbox heads, materialised nearest-neighbour FPN up-sampling -- so every algebraic rewrite of the engine (BN folding,
score-before-upsample, deconv-as-1x1 + commuted mask_score, concatenated sibling heads, fused FPN add, NHWC fc6 weight)
is checked against the formulation it replaces.  Only the state_dict KEY NAMES are shared (they are the reference's).

It is also the graph of the training-step oracle (tests/train_forward_oracle.py), which subclasses it.  Parameters are
leaf tensors in `p`, in any float dtype, on the CPU or the GPU; those named in `trainable` require grad.  Built with
the defaults, it is float32 on the CPU without gradients.  Every op is differentiable, ROIAlign included.  A subclass
freezes or plants faults through the small methods `stem_res2`, `gap` and `fcn_level`.

Reference lines restated (paths relative to /root/reference/upsnet/models/):
  resnet.py:53-100 Bottleneck, :102-153 DCNBottleneck, :155-175 conv1, :177-207 res_block, :314-356 ResNetBackbone
  fpn.py:78-104 FPN.forward            rpn.py:52-56 RPN.forward
  fcn.py:29-73 FCNSubNet, :88-108 FCNHead.forward
  rcnn.py:79-87 MaskBranch.forward, :132-146 RCNN.forward
  ../operators/modules/fpn_roi_align.py:32-62 FPNRoIAlign.forward (level = floor(2 + log2(sqrt(wh)/224 + 1e-6)) in float32)
  ../operators/modules/deform_conv.py:67-78 DeformConvWithOffset
Custom CUDA ops are replaced by torchvision's operators of the same lineage (roi_align aligned=False, sampling_ratio 2;
deform_conv2d) -- a third implementation, independent of both oracle/upsnet_oracle.c and the CUDA kernels.
"""
import numpy as np
import torch
import torch.nn.functional as F
import torchvision


class LiteralUPSNet:
    def __init__(self, state_dict, depth=(3, 4, 6, 3), num_classes=9, num_seg_classes=19, dconv_from=100, fcn_layers=2,
                 with_gap=False, with_dpyramid=False, with_dilation=False, dtype=torch.float32, device="cpu",
                 trainable=()):
        trainable = set(trainable)
        self.p = {k: v.detach().to(device=device, dtype=dtype).clone().requires_grad_(k in trainable)
                  for k, v in state_dict.items() if not k.endswith("num_batches_tracked")}
        self.depth, self.num_classes, self.num_seg_classes = depth, num_classes, num_seg_classes
        self.dconv_from, self.fcn_layers, self.with_gap = dconv_from, fcn_layers, with_gap
        self.with_dpyramid, self.with_dilation = with_dpyramid, with_dilation
        self.dtype, self.device = dtype, device

    # ------------------------------------------------------------------ primitives
    def conv(self, x, name, stride=1, padding=0, dilation=1):
        return F.conv2d(x, self.p[name + ".weight"], self.p.get(name + ".bias"), stride, padding, dilation)

    def bn(self, x, name):      # frozen BatchNorm in eval mode (resnet.py:69-78), NOT folded
        s = self.p
        return F.batch_norm(x, s[name + ".running_mean"], s[name + ".running_var"], s[name + ".weight"], s[name + ".bias"],
                            False, 0.0, 1e-5)

    def dcn(self, x, offset, wname, padding=1, dilation=1):
        return torchvision.ops.deform_conv2d(x, offset, self.p[wname + ".weight"], self.p.get(wname + ".bias"),
                                             stride=1, padding=padding, dilation=dilation)

    # ------------------------------------------------------------------ backbone
    def bottleneck(self, x, p, stride, dilation, deformable, has_down):
        out = F.relu(self.bn(self.conv(x, p + ".conv1", stride), p + ".bn1"))
        if deformable:
            offset = self.conv(out, p + ".conv2_offset", 1, 1, 1)
            out = self.dcn(out, offset, p + ".conv2", dilation, dilation)
        else:
            out = self.conv(out, p + ".conv2", 1, dilation, dilation)
        out = F.relu(self.bn(out, p + ".bn2"))
        out = self.bn(self.conv(out, p + ".conv3"), p + ".bn3")
        residual = x
        if has_down:
            residual = self.bn(self.conv(x, p + ".downsample.0", stride), p + ".downsample.1")
        return F.relu(out + residual)

    def res_block(self, x, name, blocks, stride, dilation, deformable, last_deformable):
        # resnet.py:195-203: first block, range(1, blocks - 1) middle blocks, one last block (so never fewer than two)
        n_layers = 2 + max(0, blocks - 2)
        for i in range(n_layers):
            d = deformable or (last_deformable and i == n_layers - 1)
            x = self.bottleneck(x, "resnet_backbone.%s.layers.%d" % (name, i), stride if i == 0 else 1, dilation, d, i == 0)
        return x

    def stem_res2(self, x):
        """conv1 + BN + ReLU + max-pool, then res2."""
        c1 = F.relu(self.bn(self.conv(x, "resnet_backbone.conv1.conv1", 2, 3), "resnet_backbone.conv1.bn1"))
        return self.res_block(F.max_pool2d(c1, 3, 2, 1), "res2", self.depth[0], 1, 1, False, False)

    def backbone(self, x):
        r2 = self.stem_res2(x)
        d = self.dconv_from
        r3 = self.res_block(r2, "res3", self.depth[1], 2, 1, d <= 3, self.with_dpyramid)
        r4 = self.res_block(r3, "res4", self.depth[2], 2, 1, d <= 4, self.with_dpyramid)
        s5, d5 = (1, 2) if self.with_dilation else (2, 1)
        r5 = self.res_block(r4, "res5", self.depth[3], s5, d5, d <= 5, False)
        return r2, r3, r4, r5

    # ------------------------------------------------------------------ FPN / RPN
    def gap(self, res5):
        """The global-context vector fpn_gap(GAP(res5)) (fpn.py:85) as [1, C, 1, 1]."""
        return F.linear(F.adaptive_avg_pool2d(res5, (1, 1)).flatten(1), self.p["fpn.fpn_gap.weight"],
                        self.p["fpn.fpn_gap.bias"]).view(1, -1, 1, 1)

    def fpn(self, res2, res3, res4, res5):
        up = lambda t: F.interpolate(t, scale_factor=2, mode="nearest")     # noqa: E731
        p5_1x1 = self.conv(res5, "fpn.fpn_p5_1x1")
        if self.with_gap:
            p5_1x1 = p5_1x1 + self.gap(res5)
        p4_plus = up(p5_1x1) + self.conv(res4, "fpn.fpn_p4_1x1")
        p3_plus = up(p4_plus) + self.conv(res3, "fpn.fpn_p3_1x1")
        p2_plus = up(p3_plus) + self.conv(res2, "fpn.fpn_p2_1x1")
        p2 = self.conv(p2_plus, "fpn.fpn_p2", 1, 1)
        p3 = self.conv(p3_plus, "fpn.fpn_p3", 1, 1)
        p4 = self.conv(p4_plus, "fpn.fpn_p4", 1, 1)
        p5 = self.conv(p5_1x1, "fpn.fpn_p5", 1, 1)
        p6 = F.max_pool2d(p5, 1, 2)
        return p2, p3, p4, p5, p6

    def rpn(self, feat):
        x = F.relu(self.conv(feat, "rpn.conv_proposal.0", 1, 1))
        cls_score = self.conv(x, "rpn.cls_score")
        bbox_pred = self.conv(x, "rpn.bbox_pred")
        return cls_score, bbox_pred, torch.sigmoid(cls_score)

    # ------------------------------------------------------------------ semantic head
    def fcn_level(self, x, level):
        """FCNSubNet on one FPN level; level 0 is P2."""
        for i in range(self.fcn_layers):
            p = "fcn_head.fcn_subnet.conv.%d.0" % i
            offset = self.conv(x, p + ".conv_offset", 1, 1, 1)
            x = F.relu(self.dcn(x, offset, p + ".conv"))
        return x

    def fcn_head(self, p2, p3, p4, p5, upsample_rate=4):
        outs = []
        for l, x in enumerate((p2, p3, p4, p5)):
            x = self.fcn_level(x, l)
            outs.append(x if l == 0 else F.interpolate(x, None, 2 ** l, mode="bilinear", align_corners=False))
        feat = torch.cat(outs, dim=1)
        score = self.conv(feat, "fcn_head.score")
        return {"fcn_feat": feat, "fcn_score": score,
                "fcn_output": F.interpolate(score, None, upsample_rate, mode="bilinear", align_corners=False)}

    # ------------------------------------------------------------------ roi heads
    @staticmethod
    def fpn_roi_align(feats, rois, ps):
        """[R, C, ps, ps] on the device and in the dtype of feats, differentiable in feats."""
        r = rois.detach().cpu().numpy().astype(np.float32)
        w, h = r[:, 3] - r[:, 1] + 1, r[:, 4] - r[:, 2] + 1
        lv = np.clip(np.floor(2 + np.log2(np.sqrt(w * h) / 224 + 1e-6)), 0, 3).astype(np.int64)    # fpn_roi_align.py:35-38
        if not len(lv):
            return feats[0].new_zeros((0, feats[0].shape[1], ps, ps))
        rr = rois.detach().to(feats[0].device, feats[0].dtype)
        parts, order = [], []
        for l in range(4):
            idx = np.where(lv == l)[0]
            if len(idx):
                sel = torch.from_numpy(idx).to(rr.device)
                parts.append(torchvision.ops.roi_align(feats[l], rr[sel], (ps, ps), 1.0 / 2 ** (l + 2), 2, False))
                order.append(idx)
        inv = np.argsort(np.concatenate(order))
        return torch.cat(parts)[torch.from_numpy(inv).to(rr.device)]

    def rcnn(self, feats, rois):
        x = self.fpn_roi_align(feats, rois, 7).flatten(1)
        fc6 = F.relu(F.linear(x, self.p["rcnn.fc6.0.weight"], self.p["rcnn.fc6.0.bias"]))
        fc7 = F.relu(F.linear(fc6, self.p["rcnn.fc7.0.weight"], self.p["rcnn.fc7.0.bias"]))
        return {"cls_score": F.linear(fc7, self.p["rcnn.cls_score.weight"], self.p["rcnn.cls_score.bias"]),
                "bbox_pred": F.linear(fc7, self.p["rcnn.bbox_pred.weight"], self.p["rcnn.bbox_pred.bias"]), "fc_feat": fc7}

    def mask_branch(self, feats, rois):
        x = self.fpn_roi_align(feats, rois, 14)
        for i in range(1, 5):
            x = F.relu(self.conv(x, "mask_branch.mask_conv%d.0" % i, 1, 1))
        x = F.relu(F.conv_transpose2d(x, self.p["mask_branch.mask_deconv1.0.weight"], self.p["mask_branch.mask_deconv1.0.bias"], 2))
        return self.conv(x, "mask_branch.mask_score")

    # ------------------------------------------------------------------ whole dense part
    @torch.no_grad()
    def dense(self, image):
        """image [1,3,H,W] -> dict(res, fpn (p2..p6), rpn per level, fcn_feat, fcn_score, fcn_output)."""
        res = self.backbone(image.to(self.device, self.dtype))
        p = self.fpn(*res)
        out = {"res": res, "fpn": p, "rpn": [self.rpn(f) for f in p]}
        out.update(self.fcn_head(*p[:4]))
        return out
