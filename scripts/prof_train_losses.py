"""Fused training losses (upsnet_b200.training.SemanticLoss, RPNLoss, MaskRCNNLoss), forward + backward, against the
unfused torch compositions they replace: python scripts/prof_train_losses.py [calls]

Cases, built from a seed: the semantic loss at the Cityscapes training size (fcn_score [1,19,256,512], 1024 x 2048
outputs with 255 padding); the RPN loss on RPNTargets' output for a 1024 x 2048 image (five levels, A 3, fields larger
than the maps); the Mask R-CNN loss at COCO K 81 with 512 rois and 128 mask rows.  The unfused side is the reference's
composition in plain torch (tests/train_loss_oracle.py in float32 on the device: F.interpolate + F.cross_entropy; the
per-level slices, BCE-with-logits and smooth-L1; cross-entropy, smooth-L1, the accuracy and the element-wise mask loss)
with autograd's backward.  Both sides run on the same inputs in one process and are asserted to agree first; then they
are alternated round by round after a warm-up.  Reported per call (forward + backward), as CUDA events over `calls`
calls per round: the fused op issued from Python, the fused op as replays of a CUDA graph, and the unfused composition
issued from Python; and the peak memory each side allocates above its inputs in one call, its gradients included.
The card and its power limit are read in the same run.  There is no fallback: without a GPU the script fails."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import train_loss_oracle as TL  # noqa: E402
from prof_rpn_targets import card, events_ms  # noqa: E402
from upsnet_b200 import MaskRCNNLoss, RPNLoss, SemanticLoss  # noqa: E402
from upsnet_b200.training import RPNTargets  # noqa: E402

ROUNDS = 3
DEV = torch.device("cuda", 0)


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def semantic_case():
    c = TL.semantic_case(21, 19, 256, 512, (40, 96), 0.05)
    x = t(c["fcn"]).requires_grad_(True)
    seg = t(c["seg_gt"]).long()
    mod = SemanticLoss()

    def fused(i=0):
        x.grad = None
        loss = mod(x, seg)
        loss.backward()
        return [loss.detach()], [x.grad]

    def unfused(i=0):
        x.grad = None
        loss = F.cross_entropy(F.interpolate(x, None, 4, mode="bilinear", align_corners=False), seg, ignore_index=255)
        loss.backward()
        return [loss.detach()], [x.grad]
    return fused, unfused, [x], {"S": 19, "hw": [256, 512], "outputs": [1024, 2048]}


def rpn_case():
    rng = np.random.default_rng(31)
    xy = rng.uniform(0, [1900, 950], (30, 2))
    gt = np.concatenate([xy, np.minimum(xy + rng.uniform(16, 300, (30, 2)), [2047, 1023])], 1).astype(np.float32)
    lab = RPNTargets(max_size=2048)(t(gt), 1024, 2048, seed=31)
    xs = [t((rng.standard_normal((1, 3, -(-1024 // s), -(-2048 // s))) * 2).astype(np.float32)).requires_grad_(True)
          for s in TL.STRIDES]
    ps = [t((rng.standard_normal((1, 12, -(-1024 // s), -(-2048 // s))) * 0.3).astype(np.float32)).requires_grad_(True)
          for s in TL.STRIDES]
    mod = RPNLoss(rpn_batch_size=256)

    def fused(i=0):
        for v in xs + ps:
            v.grad = None
        a, b = mod(xs, ps, lab)
        (a + b).backward()
        return [a.detach(), b.detach()], [v.grad for v in xs + ps]

    def unfused(i=0):
        for v in xs + ps:
            v.grad = None
        cls_l, box_l = 0, 0
        for x, p, s in zip(xs, ps, TL.STRIDES):
            h, w = x.shape[2:]
            sl = lambda k: lab[k % s][:, :, :h, :w]  # noqa: E731
            lb = sl("rpn_labels_fpn%d")
            cls_l = cls_l + F.binary_cross_entropy_with_logits(x, lb.float(), (lb != -1).float(), reduction="sum") / 256
            box_l = box_l + TL._smooth_l1(p, sl("rpn_bbox_targets_fpn%d"), sl("rpn_bbox_inside_weights_fpn%d"),
                                          sl("rpn_bbox_outside_weights_fpn%d"), 3.0).sum() / p.shape[0]
        (cls_l + box_l).backward()
        return [cls_l.detach(), box_l.detach()], [v.grad for v in xs + ps]
    return fused, unfused, xs + ps, {"levels": 5, "A": 3, "anchors": int(sum(x.numel() for x in xs)),
                                     "field4": list(lab["rpn_labels_fpn4"].shape[2:])}


def mask_rcnn_case():
    c = TL.mask_rcnn_case(45, 512, 81, 128)
    inp = [t(c[k]) for k in TL.NAMES]
    for v in inp[:3]:
        v.requires_grad_(True)
    mod = MaskRCNNLoss()

    def fused(i=0):
        for v in inp[:3]:
            v.grad = None
        out = mod(*inp)
        (out[0] + out[1] + out[2]).backward()
        return [v.detach() for v in out], [v.grad for v in inp[:3]]

    def unfused(i=0):
        x, p, m, lab, bt, biw, bow, mt = inp
        for v in inp[:3]:
            v.grad = None
        cls_loss = F.cross_entropy(x, lab, ignore_index=-1)
        bbox = TL._smooth_l1(p, bt, biw, bow, 1.0)
        bbox_loss = bbox.sum() / bbox.shape[0]
        with torch.no_grad():
            ignore = (lab == -1).long().sum()
            acc = ((x.max(1)[1] == lab).long().sum() - ignore).float() / (lab.shape[0] - ignore).float()
        tt = mt.view(m.shape)
        wgt = (tt != -1).float()
        b = (m >= 0).float()
        mask_loss = ((-m * (tt - b) + torch.log(1 + torch.exp(m - 2 * m * b))) * wgt).sum() / (wgt.sum() + 1e-10)
        (cls_loss + bbox_loss + mask_loss).backward()
        return [cls_loss.detach(), bbox_loss.detach(), mask_loss.detach(), acc], [v.grad for v in inp[:3]]
    return fused, unfused, inp[:3], {"R": 512, "K": 81, "mask_rows": 128}


def peak_mb(fn, leaves):
    """MB allocated above the inputs during one call, the gradients it leaves included."""
    fn()
    for v in leaves:
        v.grad = None
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)


def measure(name, build, n_calls):
    fused, unfused, leaves, info = build()
    lf, gf = fused()
    lf, gf = [v.clone() for v in lf], [v.clone() for v in gf]
    lu, gu = unfused()
    for a, b in zip(lf, lu):
        assert abs(float(a) - float(b)) <= 1e-5 * abs(float(b)) + 1e-7, (name, float(a), float(b))
    # the unfused float32 backward is not deterministic (the up-sampling backward adds with atomics): its largest
    # difference from the fused gradient is reported, and only a gross disagreement fails
    grad_diff = max(float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30) for a, b in zip(gf, gu))
    assert grad_diff <= 1e-3, (name, grad_diff)
    mem = {"fused": peak_mb(fused, leaves), "unfused": peak_mb(unfused, leaves)}
    for _ in range(5):
        fused(); unfused()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fused()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fused()
    graph.replay()
    torch.cuda.synchronize()
    tm = {"fused_issued": [], "fused_graph": [], "unfused_issued": []}
    for _ in range(ROUNDS):
        tm["fused_issued"].append(events_ms(fused, n_calls))
        tm["unfused_issued"].append(events_ms(unfused, n_calls))
        tm["fused_graph"].append(events_ms(lambda i: graph.replay(), n_calls))
    return dict(case=name, **info, losses=[round(float(v), 6) for v in lf],
                ms_per_call={k: [round(v, 4) for v in vs] for k, vs in tm.items()}, peak_mb_per_call=mem,
                grad_max_diff_over_max=float("%.3g" % grad_diff),
                calls_per_round=n_calls, rounds=ROUNDS)


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    assert torch.cuda.is_available(), "needs cuda:0"
    res = {"card": card(), "cases": [measure("semantic_cityscapes", semantic_case, n), measure("rpn_1024x2048", rpn_case, n),
                                     measure("mask_rcnn_coco", mask_rcnn_case, n)]}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
