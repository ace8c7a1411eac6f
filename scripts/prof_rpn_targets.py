"""Device RPN training targets (upsnet_rpn_targets) per image: python scripts/prof_rpn_targets.py [calls]

The four full-size cases of tests/rpn_target_oracle.FULL (COCO 800x1333 with 15 / 90 boxes, Cityscapes 1024x2048 with
50 / 300 boxes, built from a seed).  Reports the per-image device time as CUDA events over many calls issued one by one
from Python and over replays of a CUDA graph of the calls, the numpy oracle's host time for one image, and the card and
its power limit, read in the same run."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import rpn_target_oracle as RO  # noqa: E402
from upsnet_b200.training import RPNTargets  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        out = "nvidia-smi unavailable (%s)" % e
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q + ": " + out}


def events_ms(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(n):
        fn(i)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def measure(name, n_calls):
    dev = torch.device("cuda", 0)
    entry, scale, cfg = RO.full_case(name, 0)
    t = RPNTargets(max_size=cfg.max_size)
    gt, h, w = RO.gt_from_roidb(entry, scale)
    g = torch.from_numpy(gt).to(dev)

    def call(i=0):
        return t(g, h, w, seed=i)

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
    ref = RO.rpn_targets(gt, h, w, cfg, 0)
    host = (time.perf_counter() - t0) * 1e3
    return {"case": name, "G": int(gt.shape[0]), "anchors": t.num_anchors, "inside": int(ref["counts"][0]),
            "device_ms_issued": round(issued, 4), "device_ms_graph": round(replay, 4), "oracle_host_ms": round(host, 1),
            "calls": n_calls}


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    assert torch.cuda.is_available(), "needs cuda:0"
    res = {"card": card(), "cases": [measure(c[0], n) for c in RO.FULL]}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
