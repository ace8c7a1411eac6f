"""Device Mask R-CNN proposal targets (upsnet_proposal_targets) per image: python scripts/prof_proposal_targets.py [calls]

The full-size cases of tests/proposal_target_oracle.FULL (COCO 800x1333 with 2000 proposals and 15 / 90 objects, K = 81;
Cityscapes 1024x2048 with 2000 proposals and 50 objects, K = 9; built from a seed).  Reports the per-image device time
as CUDA events over many calls issued one by one from Python and over replays of a CUDA graph of the call (the packed
ground truth uploaded once), the numpy oracle's host time for one image, and the card and its power limit, read in the
same run."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import proposal_target_oracle as PO  # noqa: E402
from prof_rpn_targets import card, events_ms  # noqa: E402
from upsnet_b200.training import ProposalTargets  # noqa: E402


def measure(name, n_calls):
    dev = torch.device("cuda", 0)
    e, rois, scale, cfg = PO.full_case(name, 0)
    t = ProposalTargets(num_classes=cfg.num_classes)
    r = torch.from_numpy(rois).to(dev)
    pk = t.pack_roidb(e, dev)

    def call(i=0):
        return t(r, pk, scale, seed=i)

    for i in range(5):
        call(i)
    torch.cuda.synchronize()
    issued = events_ms(call, n_calls)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call()
    graph.replay()
    torch.cuda.synchronize()
    replay = events_ms(lambda i: graph.replay(), n_calls)
    t0 = time.perf_counter()
    ref = PO.proposal_targets(rois, e, scale, cfg, 0)
    host = (time.perf_counter() - t0) * 1e3
    return {"case": name, "K": cfg.num_classes, "objects": int(pk.O), "rois": int(rois.shape[0]),
            "fg": int(ref["counts"][0]), "device_ms_issued": round(issued, 4), "device_ms_graph": round(replay, 4),
            "oracle_host_ms": round(host, 1), "calls": n_calls}


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    assert torch.cuda.is_available(), "needs cuda:0"
    res = {"card": card(), "cases": [measure(c[0], n) for c in PO.FULL]}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
