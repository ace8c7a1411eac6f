"""Fused panoptic loss (upsnet_b200.training.PanopticLoss), forward + backward, against the unfused composition it
replaces: python scripts/prof_panoptic_loss.py [calls]

Cases (tests/panoptic_loss_oracle.FULL, built from a seed): Cityscapes (S 19, 256x512, k 35) and COCO (S 133, 200x336,
k 10 and k 63).  The unfused side is what a user of this package writes without the fused op: SegTerm + MaskTerm +
MaskMatching + the void logits + torch.cat + F.cross_entropy + the accuracy, with autograd's backward.  Both sides run
on the same inputs in one process, alternated round by round after a warm-up; the two are asserted to agree before
anything is timed.  Reported per call (forward + backward), as CUDA events over `calls` calls per round: the fused op
issued from Python, the fused op as replays of a CUDA graph, the unfused composition issued from Python (it reads the
device back three times per call and cannot be captured); and the card and its power limit, read in the same run.
There is no fallback: without a GPU the script fails."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import panoptic_loss_oracle as PL  # noqa: E402
from prof_rpn_targets import card, events_ms  # noqa: E402
from upsnet_b200 import MaskMatching, MaskTerm, PanopticLoss, SegTerm  # noqa: E402

ROUNDS = 3


def measure(name, n_calls):
    dev = torch.device("cuda", 0)
    c = PL.case(PL.FULL[name])
    S, nc = c["fcn"].shape[1], c["num_classes"]
    fcn, ms, rois, cls, seg, mgt, keep = (torch.from_numpy(np.ascontiguousarray(c[k_])).to(dev) for k_ in
                                          ("fcn", "mask_score", "rois", "cls", "seg_gt", "mask_gt", "keep"))
    fcn.requires_grad_(True); ms.requires_grad_(True)
    fused_mod = PanopticLoss(num_seg_classes=S, num_classes=nc)
    seg_term, mask_term, matching = SegTerm(S, num_classes=nc), MaskTerm(S, num_classes=nc), MaskMatching(S, True, num_classes=nc)
    mgt64 = mgt.long()

    def fused(i=0):
        fcn.grad = ms.grad = None
        loss, acc = fused_mod(fcn, ms, rois, cls, seg, mgt, keep)
        loss.backward()
        return loss.detach(), acc

    def unfused(i=0):
        fcn.grad = ms.grad = None
        sel = ms.gather(1, cls.view(-1, 1, 1, 1).expand(-1, -1, 28, 28))
        seg_logits, seg_inst = seg_term(cls, fcn, rois)
        mask_logits = mask_term(sel, rois, cls, fcn)
        void = fcn[:, S - nc + 1:].max(1, keepdim=True)[0] - seg_inst.max(1, keepdim=True)[0]
        logits = torch.cat([seg_logits, seg_inst + mask_logits, void], 1)
        with torch.no_grad():
            gt = matching(seg, mgt64, keep)
            correct = (logits.max(1)[1].view(-1) == gt.view(-1)).sum()
            acc = correct.float() / (gt.numel() - (gt == 255).sum()).float()
        loss = torch.nn.functional.cross_entropy(logits, gt, ignore_index=255, reduction="none").mean()
        loss.backward()
        return loss.detach(), acc

    lf, af = fused()
    gf = (fcn.grad.clone(), ms.grad.clone())
    lu, au = unfused()
    assert abs(float(lf) - float(lu)) <= 1e-5 * abs(float(lu)) and abs(float(af) - float(au)) <= 1e-3
    for a, b in zip(gf, (fcn.grad, ms.grad)):
        assert float((a - b).abs().max()) <= 2e-5 * float(b.abs().max())
    for i in range(5):
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
    t = {"fused_issued": [], "fused_graph": [], "unfused_issued": []}
    for _ in range(ROUNDS):
        t["fused_issued"].append(events_ms(fused, n_calls))
        t["unfused_issued"].append(events_ms(unfused, n_calls))
        t["fused_graph"].append(events_ms(lambda i: graph.replay(), n_calls))
    h, w = fcn.shape[2:]
    return {"case": name, "S": S, "hw": [int(h), int(w)], "k": int(ms.shape[0]), "loss": round(float(lf), 6),
            "ms_per_call": {k_: [round(v, 4) for v in vs] for k_, vs in t.items()},
            "calls_per_round": n_calls, "rounds": ROUNDS}


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 100
    assert torch.cuda.is_available(), "needs cuda:0"
    res = {"card": card(), "cases": [measure(name, n) for name in ("cityscapes", "coco_k10", "coco_k63")]}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
