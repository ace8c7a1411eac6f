"""Times the semantic head's ROI loss, forward + backward, at COCO size (S 133, fcn_score 200x336, R 15 and 90): the
fused FcnRoiLoss, issued from Python and replayed from a CUDA graph, against the unfused composition the reference
runs (x2/x4/x8 bilinear up-sampling, the 512-channel concat, torchvision's roi_align(aligned=False, sampling_ratio=2),
the 1x1 score conv, the cross-entropy, autograd), with the peak memory each adds above its inputs.
Run: python scripts/prof_fcn_roi_loss.py  (needs an H100; prints one JSON line)."""
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def timed(fn, iters=50, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def peak(fn):
    fn()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def main():
    from torchvision.ops import roi_align
    import fcn_roi_loss_oracle as O
    from upsnet_b200 import FcnRoiLoss
    dev = torch.device("cuda", 0)
    S, h, w = 133, 200, 336
    g = torch.Generator().manual_seed(0)
    levels = [torch.randn(1, 128, h >> l, w >> l, generator=g).to(dev).requires_grad_(True) for l in range(4)]
    weight = (torch.randn(S, 512, 1, 1, generator=g) * 0.05).to(dev).requires_grad_(True)
    bias = torch.randn(S, generator=g).to(dev).requires_grad_(True)
    fcn = (torch.randn(1, S, h, w, generator=g) * 3).to(dev).requires_grad_(True)
    res = {}
    for R in (15, 90):
        rois = O.boxes(g, R, h, w, "random").to(dev)
        seg = torch.randint(0, S, (R, 28, 28), generator=g).to(dev)
        m = FcnRoiLoss(28)

        def fused():
            fcn.grad = bias.grad = None
            m(fcn, bias, rois, seg).backward()

        def unfused():
            for t in levels + [weight, bias]:
                t.grad = None
            p2, p3, p4, p5 = levels
            up = lambda t, f: F.interpolate(t, None, f, mode="bilinear", align_corners=False)  # noqa: E731
            feat = torch.cat([p2, up(p3, 2), up(p4, 4), up(p5, 8)], 1)
            score = F.conv2d(roi_align(feat, rois, (28, 28), 0.25, 2, aligned=False), weight, bias)
            F.cross_entropy(score, seg, ignore_index=255, reduction="none").mean().backward()

        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            fused()
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            fused()
        res["R%d" % R] = {"fused_ms": timed(fused), "fused_graph_ms": timed(graph.replay), "unfused_ms": timed(unfused),
                          "fused_peak_mb": peak(fused), "unfused_peak_mb": peak(unfused)}
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(json.dumps({"card": card, "S": S, "fcn_score": [h, w], "results": res}))


if __name__ == "__main__":
    main()
