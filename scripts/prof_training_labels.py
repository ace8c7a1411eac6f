"""Device panoptic training labels (upsnet_training_labels) per image: python scripts/prof_training_labels.py [calls]

The full-size cases of tests/label_oracle.FULL (Cityscapes 1024x2048 with 50 / 300 instances, COCO 800x1333 with 15 /
90, built from a seed; seg_roi_gt on).  Reports the per-image device time as CUDA events over replays of a CUDA graph
of the launch (tables and polygons uploaded once) and over whole calls issued one by one from Python (host tables,
their upload and the launch), the byte floor of the outputs (uint8 mask_gt), the numpy oracle's host time for one
image, and the card and its power limit, read in the same run."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch  # noqa: E402

import label_oracle as LO  # noqa: E402
from prof_rpn_targets import card, events_ms  # noqa: E402
from upsnet_b200.training import PanopticLabels  # noqa: E402


def measure(name, n_calls):
    dev = torch.device("cuda", 0)
    e, lab, im_shape, scale, dataset = LO.full_case(name)
    L = PanopticLabels(dataset=dataset, with_roi=True)
    pk = L.pack_roidb(e, scale, dev)
    labd = torch.from_numpy(lab).to(dev)
    tab = L.prepare(tuple(labd.shape), pk, im_shape, scale, e["flipped"], dev)

    def call(i=0):
        return L(labd, pk, im_shape, scale, e["flipped"])

    out = call()
    torch.cuda.synchronize()
    issued = events_ms(call, n_calls)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        L.launch(labd, pk, tab)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        L.launch(labd, pk, tab)
    graph.replay()
    torch.cuda.synchronize()
    replay = events_ms(lambda i: graph.replay(), n_calls)
    floor = sum(v.numel() * v.element_size() for v in out.values()) + lab.size
    t0 = time.perf_counter()
    LO.labels(e, lab, im_shape, scale, dataset, True)
    host = (time.perf_counter() - t0) * 1e3
    return {"case": name, "G": int(pk.G), "out_shapes": {k: list(v.shape) for k, v in out.items()},
            "byte_floor_MB": round(floor / 1e6, 2), "floor_ms_at_3.35TBs": round(floor / 3.35e9, 4),
            "device_ms_graph": round(replay, 4), "device_ms_issued": round(issued, 4),
            "oracle_host_ms": round(host, 1), "calls": n_calls}


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    assert torch.cuda.is_available(), "needs cuda:0"
    res = {"card": card(), "cases": [measure(c[0], n) for c in LO.FULL]}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
