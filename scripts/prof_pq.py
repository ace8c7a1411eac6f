"""Device PQ statistics (upsnet_pq_update) and label-map restore (upsnet_label_restore) at 1024x2048 with
Cityscapes-like segment counts: python scripts/prof_pq.py [images]

Reports the per-image device time (CUDA events over many images after warm-up; once as issued by update() from Python,
once replaying a CUDA graph of the updates, which removes the host issue time), the bytes each pass must move against
the H100 SXM HBM3 floor of 3.35 TB/s, the numpy oracle's host time for one image, and the card and its power limit."""
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

import upsnet_b200 as U  # noqa: E402
import pq_oracle as P  # noqa: E402
from test_gpu_pq import CATS, random_case  # noqa: E402

HBM = 3.35e12


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


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(1)
    H, W = 1024, 2048
    imgs = [random_case(rng, H, W, n_gt=60, n_pred=40) for _ in range(4)]       # ~70 gt, ~80-100 prediction segments
    dimgs = [(torch.from_numpy(p).to(dev), torch.from_numpy(g).to(dev), s) for p, g, s in imgs]
    pq = U.PanopticQuality(CATS)
    for i in range(8):
        pq.update(*dimgs[i % 4])
    pq.check_errors()
    torch.cuda.synchronize()
    issued = events_ms(lambda i: pq.update(*dimgs[i % 4]), n)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        pq.update(*dimgs[0])
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        for d in dimgs:
            pq.update(*d)
    graph = events_ms(lambda i: g.replay(), max(1, n // 4)) / 4
    pq.check_errors()
    segs = [len(s_) for _, _, s_ in imgs]
    npred = [len(np.unique(p[..., 0].astype(np.int64) * 256 + p[..., 1])) for p, _, _ in imgs]

    lab = [torch.from_numpy(rng.integers(0, 30, (1, H, W))).to(dev) for _ in range(2)]
    info = np.array([H, W, 1.0], np.float32)
    for _ in range(5):
        U.label_restore(lab[0], info, lab[1])
    torch.cuda.synchronize()
    restore = events_ms(lambda i: U.label_restore(lab[0], info, lab[1]), n)
    coco = [torch.from_numpy(rng.integers(0, 30, (1, 1344, 1344))).to(dev) for _ in range(2)]
    cinfo = np.array([800, 1333, 1.0], np.float32)        # 800x1333 input in a 1344-padded map, restored at scale 1
    cinfo[2] = np.float32(800.0 / 640.0)                   # original 640x1066 image
    U.label_restore(coco[0], cinfo, coco[1])
    torch.cuda.synchronize()
    restore_coco = events_ms(lambda i: U.label_restore(coco[0], cinfo, coco[1]), n)
    oh, ow = P.label_restore(np.zeros((1344, 1344), np.int64), cinfo).shape

    t0 = time.perf_counter()
    P.pq_image(*imgs[0], CATS)
    host = (time.perf_counter() - t0) * 1e3

    px = H * W
    rep = {
        "card": card(),
        "images": n, "H": H, "W": W, "gt_segments": segs, "pred_class_instance_pairs_incl_void": npred,
        "pq_update_ms_issued_from_python": round(issued, 4),
        "pq_update_ms_graph_replay": round(graph, 4),
        "pq_pixel_pass_bytes": 6 * px, "pq_pixel_pass_floor_ms": round(6 * px / HBM * 1e3, 4),
        "label_restore_pair_ms_1024x2048": round(restore, 4),
        "label_restore_bytes_1024x2048": 32 * px, "label_restore_floor_ms_1024x2048": round(32 * px / HBM * 1e3, 4),
        "label_restore_pair_ms_coco_1344_to_%dx%d" % (oh, ow): round(restore_coco, 4),
        "oracle_host_ms_one_image": round(host, 1),
    }
    print(json.dumps(rep, indent=1))


if __name__ == "__main__":
    main()
