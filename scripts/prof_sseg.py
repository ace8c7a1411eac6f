"""Device semantic-segmentation confusion matrix (upsnet_sseg_update through SegmentationIoU.update) at 1024x2048 with
C = 19 (Cityscapes) and at a COCO size with C = 133: python scripts/prof_sseg.py [images]

Reports the per-image device time (CUDA events over many images after warm-up; once as issued by update() from Python,
once replaying a CUDA graph of the updates, which removes the host issue time) for int64 and uint8 predictions, the
bytes the pass must move (gt 1 B + one prediction element per pixel) against the H100 SXM HBM3 floor of 3.35 TB/s, the
numpy oracle's host time for one image, and the card and its power limit."""
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
import sseg_oracle as S  # noqa: E402

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


def measure(C, H, W, n, dev):
    imgs = [S.synthetic_case(k, H, W, C) for k in range(4)]
    out = {}
    for dtype in (np.int64, np.uint8):
        d = [(torch.from_numpy(p.astype(dtype)).to(dev), torch.from_numpy(g).to(dev)) for p, g in imgs]
        miou = U.SegmentationIoU(C)
        for i in range(8):
            miou.update(*d[i % 4])
        torch.cuda.synchronize()
        issued = events_ms(lambda i: miou.update(*d[i % 4]), n)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            miou.update(*d[0])
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for x in d:
                miou.update(*x)
        for _ in range(3):
            g.replay()
        torch.cuda.synchronize()
        graph = events_ms(lambda i: g.replay(), max(1, n // 4)) / 4
        miou.reset()
        miou.update(*d[0])
        assert np.array_equal(miou.confusion_matrix(), S.confusion(*imgs[0], C))       # the timed path computes the oracle's matrix
        bpp = 1 + np.dtype(dtype).itemsize
        name = np.dtype(dtype).name
        out[name] = {"update_ms_issued_from_python": round(issued, 4), "update_ms_graph_replay": round(graph, 4),
                     "bytes": bpp * H * W, "floor_ms": round(bpp * H * W / HBM * 1e3, 4)}
    t0 = time.perf_counter()
    S.confusion(*imgs[0], C)
    out["oracle_host_ms_one_image"] = round((time.perf_counter() - t0) * 1e3, 1)
    return out


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 400
    dev = torch.device("cuda", 0)
    rep = {"card": card(), "images": n,
           "cityscapes_1024x2048_C19": measure(19, 1024, 2048, n, dev),
           "coco_800x1333_C133": measure(133, 800, 1333, n, dev)}
    print(json.dumps(rep, indent=1))


if __name__ == "__main__":
    main()
