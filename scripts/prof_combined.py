"""Device combined panoptic result (upsnet_combined_pan_result) per image: python scripts/prof_combined.py [calls]

Two sizes: 1024x2048 with Cityscapes class counts (19 / 9) and 800x1333 with COCO's (133 / 81), about 100 detections each
(tests/combined_oracle.py builds them from a seed).  Reports the per-image device time three ways -- CUDA events over
many calls issued one by one from Python, CUDA events over replays of a CUDA graph of the calls (no host issue time),
and the numpy oracle on the host for one image -- plus how many detections passed the score test and were kept, and the
card and its power limit, read in the same run."""
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

import combined_oracle as CO  # noqa: E402
from upsnet_b200 import operators as ops  # noqa: E402


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


def measure(name, sem, scores, cls, runs, nsc, nc, n_calls):
    dev = torch.device("cuda", 0)
    cn, rl = CO.pack_runs(runs)
    args = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (sem.astype(np.int64), scores, cls, cn.view(np.int32), rl)]
    sem_d, sc_d, cl_d, cn_d, rl_d = args

    def call(i=0):
        return ops.combined_pan_result(sem_d, sc_d, cl_d, (cn_d, rl_d), nsc, nc, check_errors=False)

    out = ops.combined_pan_result(sem_d, sc_d, cl_d, (cn_d, rl_d), nsc, nc)           # checks the error word once
    for _ in range(5):
        call()
    torch.cuda.synchronize()
    issued = events_ms(call, n_calls)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(4):
            call()
    g.replay()
    torch.cuda.synchronize()
    graph = events_ms(lambda i: g.replay(), max(1, n_calls // 4)) / 4
    t0 = time.perf_counter()
    want = CO.combined_pan_result(sem, scores, cls, runs, nsc, nc)
    host = (time.perf_counter() - t0) * 1e3
    pan = out.cpu().numpy()
    assert np.array_equal(pan, want), name
    kept = len({(int(a), int(b)) for a, b in pan[pan[..., 1] > 0][:, :2]})
    H, W = sem.shape
    return {"size": "%dx%d" % (H, W), "num_seg_classes": nsc, "num_classes": nc, "detections": len(runs),
            "score_ge_0.6": int((scores >= np.float32(0.6)).sum()), "kept_instances": kept,
            "ms_graph_replay": round(graph, 4), "ms_issued_from_python": round(issued, 4),
            "ms_numpy_oracle_host": round(host, 1), "matches_oracle": True}


def main():
    n_calls = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    rep = {"card": card(), "calls": n_calls}
    sem, scores, cls, runs = CO.large_case()
    rep["cityscapes_1024x2048"] = measure("cityscapes", sem, scores, cls, runs, 19, 9, n_calls)
    rng = np.random.default_rng(800)
    sem = CO.semantic_map(rng, 800, 1333, 133, block=32)
    scores, cls, runs = CO.random_detections(rng, 800, 1333, 100, 81)
    rep["coco_800x1333"] = measure("coco", sem, scores, cls, runs, 133, 81, n_calls)
    print(json.dumps(rep, indent=1))


if __name__ == "__main__":
    main()
