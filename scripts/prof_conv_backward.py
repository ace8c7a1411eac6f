"""Per-layer timing of the dense-conv backward (csrc/conv_backward.cu via upsnet_b200.training.conv2d_backward) over
the trainable dense layers of UPSNet-50 at 1024x2048 (Cityscapes, backbone_freeze_at = 2: res3-res5 without the
deformable res5 3x3, FPN, RPN head over P2-P6, fc6 / fc7 / cls / bbox on 512 rois, the mask branch on 163 rois),
next to torch's conv backward (cuDNN: fp32 with TF32 off, TF32 on, bf16) in the same process, rounds alternated.

Each variant is captured in a CUDA graph and timed by events over `--iters` replays; the median of `--rounds` rounds is
reported.  Ours: prepare (dY -> g, d bias, d residual), dgrad = (prepare + dX) - prepare, wgrad = (prepare + dW) -
prepare.  Torch: conv2d_input + conv2d_weight + the bias sum.  TFLOP/s are algorithmic (2 P Cout Cin k^2 per gradient);
mma_frac is the issued tensor-core rate (x3 for bf16x3) over the 989 TFLOP/s dense-bf16 data-sheet peak.
Prints one row per layer, totals, the card name and its power limit.  `python scripts/prof_conv_backward.py`."""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from upsnet_b200 import _lib, training  # noqa: E402
from upsnet_b200 import operators as ops  # noqa: E402

PEAK_BF16 = 989e12


def layers():
    """(name, count, N, Cin, H, W, Cout, k, stride, pad, relu, residual) at 1024x2048: P2 = 256x512."""
    L = []
    # res3 (256x512 -> 128x256), 4 blocks
    L += [("res3.0 conv1 1x1 s2", 1, 1, 256, 256, 512, 128, 1, 2, 0, True, None),
          ("res3.0 downsample s2", 1, 1, 256, 256, 512, 512, 1, 2, 0, False, None),
          ("res3 conv2 3x3", 4, 1, 128, 128, 256, 128, 3, 1, 1, True, None),
          ("res3 conv3 1x1 +res", 4, 1, 128, 128, 256, 512, 1, 1, 0, True, "same"),
          ("res3 conv1 1x1", 3, 1, 512, 128, 256, 128, 1, 1, 0, True, None)]
    # res4 (-> 64x128), 6 blocks
    L += [("res4.0 conv1 1x1 s2", 1, 1, 512, 128, 256, 256, 1, 2, 0, True, None),
          ("res4.0 downsample s2", 1, 1, 512, 128, 256, 1024, 1, 2, 0, False, None),
          ("res4 conv2 3x3", 6, 1, 256, 64, 128, 256, 3, 1, 1, True, None),
          ("res4 conv3 1x1 +res", 6, 1, 256, 64, 128, 1024, 1, 1, 0, True, "same"),
          ("res4 conv1 1x1", 5, 1, 1024, 64, 128, 256, 1, 1, 0, True, None)]
    # res5 (-> 32x64), 3 blocks; the 3x3 is deformable (not a dense layer)
    L += [("res5.0 conv1 1x1 s2", 1, 1, 1024, 64, 128, 512, 1, 2, 0, True, None),
          ("res5.0 downsample s2", 1, 1, 1024, 64, 128, 2048, 1, 2, 0, False, None),
          ("res5 conv3 1x1 +res", 3, 1, 512, 32, 64, 2048, 1, 1, 0, True, "same"),
          ("res5 conv1 1x1", 2, 1, 2048, 32, 64, 512, 1, 1, 0, True, None)]
    # FPN: laterals (+ top-down residual_up2), 3x3 outputs
    L += [("fpn_lat2 +up2", 1, 1, 256, 256, 512, 256, 1, 1, 0, False, "up2"),
          ("fpn_lat3 +up2", 1, 1, 512, 128, 256, 256, 1, 1, 0, False, "up2"),
          ("fpn_lat4 +up2", 1, 1, 1024, 64, 128, 256, 1, 1, 0, False, "up2"),
          ("fpn_lat5", 1, 1, 2048, 32, 64, 256, 1, 1, 0, False, None),
          ("fpn_p2 3x3", 1, 1, 256, 256, 512, 256, 3, 1, 1, False, None),
          ("fpn_p3 3x3", 1, 1, 256, 128, 256, 256, 3, 1, 1, False, None),
          ("fpn_p4 3x3", 1, 1, 256, 64, 128, 256, 3, 1, 1, False, None),
          ("fpn_p5 3x3", 1, 1, 256, 32, 64, 256, 3, 1, 1, False, None)]
    # RPN head, shared over P2..P6
    for lv, (h, w) in enumerate([(256, 512), (128, 256), (64, 128), (32, 64), (16, 32)]):
        L += [("rpn 3x3 P%d" % (lv + 2), 1, 1, 256, h, w, 256, 3, 1, 1, True, None),
              ("rpn cls+bbox P%d" % (lv + 2), 1, 1, 256, h, w, 15, 1, 1, 0, False, None)]
    # RCNN box head on 512 rois, mask branch on 163 rois
    L += [("fc6 12544->1024", 1, 512, 12544, 1, 1, 1024, 1, 1, 0, True, None),
          ("fc7 1024->1024", 1, 512, 1024, 1, 1, 1024, 1, 1, 0, True, None),
          ("cls+bbox 9+36", 1, 512, 1024, 1, 1, 45, 1, 1, 0, False, None),
          ("mask conv 3x3", 4, 163, 256, 14, 14, 256, 3, 1, 1, True, None),
          ("mask deconv 2x2", 1, 163, 256, 14, 14, 1024, 1, 1, 0, True, None),
          ("mask score 9", 1, 163, 256, 28, 28, 9, 1, 1, 0, False, None)]
    return L


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                                        # noqa: BLE001
        out = "power limit unknown"
    return "%s (%s)" % (name, out)


def graphed(fn):
    """(graph, fn): the closure is returned with the graph because it holds the graph's input tensors -- entering a
    capture empties torch's allocator cache, so an input freed before a replay may be unmapped by the next capture."""
    fn()
    fn()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            fn()
    torch.cuda.synchronize()
    return g, fn


def time_graph(gf, iters):
    g = gf[0]
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--only", default="", help="substring filter on the layer names")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "prof_conv_backward needs a GPU"
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    print("card: %s" % card())
    cols = ["prep", "dgrad", "wgrad"]
    hdr = "%-22s %3s %9s | %-37s | %-37s | %8s %8s %8s" % ("layer", "n", "GFLOP/gr", "bf16: prep dgrad wgrad ms (TF/s mma)",
                                                           "bf16x3: prep dgrad wgrad ms (TF/s mma)", "cudnn32", "tf32", "cudnnbf")
    print(hdr)
    tot = {}
    for name, cnt, N, Cin, H, W, Cout, k, s, p, relu, res in layers():
        if args.only and args.only not in name:
            continue
        Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
        x = torch.randn((N, Cin, H, W), device=dev)
        w = torch.randn((Cout, Cin, k, k), device=dev) * (2.0 / (Cin * k * k)) ** 0.5
        bias = torch.randn((Cout,), device=dev) * 0.1
        dy = torch.randn((N, Cout, Ho, Wo), device=dev)
        flop = 2.0 * N * Ho * Wo * Cout * Cin * k * k          # per gradient (dX or dW)
        graphs = {}
        for prec_name, prec in (("bf16", _lib.PREC_BF16), ("bf16x3", _lib.PREC_BF16X3)):
            xs = training._stored_input(x, prec)
            y = ops.conv2d(training._kernel_input(xs, prec), w, bias, s, p, 1, relu=relu, precision=prec,
                           out_dtype=torch.float32)
            ys = y.permute(0, 2, 3, 1)
            geom = (N, Cin, H, W, (s, s), (p, p), (1, 1))
            up2 = res == "up2"
            for part, need in (("p", (False, False, True, res is not None)), ("px", (True, False, True, res is not None)),
                               ("pw", (False, True, True, res is not None))):
                graphs[(prec_name, part)] = graphed(
                    lambda xs=xs, ys=ys, prec=prec, need=need, up2=up2: training.conv2d_backward(
                        dy, xs, ys, w, geom, prec, relu, True, up2, need))
        # torch's backward: dX + dW + bias sum per dtype
        tvars = {}
        for tname, dt, tf32 in (("cudnn32", torch.float32, False), ("tf32", torch.float32, True),
                                ("cudnnbf", torch.bfloat16, False)):
            xt, wt, dyt = x.to(dt), w.to(dt), dy.to(dt)

            def tb(xt=xt, wt=wt, dyt=dyt, tf32=tf32):
                torch.backends.cudnn.allow_tf32 = tf32
                torch.nn.grad.conv2d_input(xt.shape, wt, dyt, stride=s, padding=p)
                torch.nn.grad.conv2d_weight(xt, wt.shape, dyt, stride=s, padding=p)
                dyt.sum((0, 2, 3))
            torch.backends.cudnn.allow_tf32 = tf32
            tvars[tname] = (graphed(tb), tf32)
        times = {key: [] for key in list(graphs) + list(tvars)}
        for _ in range(args.rounds):
            for key, g in graphs.items():
                times[key].append(time_graph(g, args.iters))
            for key, (g, tf32) in tvars.items():
                times[key].append(time_graph(g, args.iters))
        med = {key: sorted(v)[len(v) // 2] for key, v in times.items()}
        cells = []
        for prec_name, passes in (("bf16", 1), ("bf16x3", 3)):
            pr = med[(prec_name, "p")]
            dg = max(med[(prec_name, "px")] - pr, 1e-6)
            wg = max(med[(prec_name, "pw")] - pr, 1e-6)
            rate = 2 * flop / ((dg + wg) * 1e-3)
            cells.append("%6.3f %6.3f %6.3f (%5.0f %4.2f)" % (pr, dg, wg, rate / 1e12, rate * passes / PEAK_BF16))
            for key, v in ((prec_name + " prep", pr), (prec_name + " dgrad", dg), (prec_name + " wgrad", wg)):
                tot[key] = tot.get(key, 0.0) + cnt * v
        for key in ("cudnn32", "tf32", "cudnnbf"):
            tot[key] = tot.get(key, 0.0) + cnt * med[key]
        print("%-22s %3d %9.2f | %-37s | %-37s | %8.3f %8.3f %8.3f" % (
            name, cnt, flop / 1e9, cells[0], cells[1], med["cudnn32"], med["tf32"], med["cudnnbf"]))
        del graphs, tvars
        torch.cuda.empty_cache()
    torch.backends.cudnn.allow_tf32 = True
    print("totals (ms, layer times x count):")
    for key in sorted(tot):
        print("  %-14s %8.3f" % (key, tot[key]))
    print("  bf16 backward   %8.3f   bf16x3 backward %8.3f" % (
        tot.get("bf16 prep", 0) + tot.get("bf16 dgrad", 0) + tot.get("bf16 wgrad", 0),
        tot.get("bf16x3 prep", 0) + tot.get("bf16x3 dgrad", 0) + tot.get("bf16x3 wgrad", 0)))
    print("card: %s" % card())


if __name__ == "__main__":
    main()
