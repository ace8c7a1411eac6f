"""CUDA-event timer for the TMA-fed dense conv kernel (csrc/igemm_tma.cu) at the layer shapes the model runs (Cityscapes
1024x2048 input, ResNet-50-FPN): the bf16 activation stream, and the hi/lo pair stream (precision bf16x3) with each
output-channel tile forced through upsnet_tma_set_tile_n.  One line per layer and mode: ms per call, algorithmic TFLOP/s
(2 * P * Cout * Cin * k * k) and executed TFLOP/s (the pair stream issues three bf16 tensor-core passes per algorithmic
flop).  A forced tile that does not fit runs at the tile the launcher falls back to.
Usage: python scripts/prof_tma.py [--reps 20]"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import upsnet_b200 as U
from upsnet_b200 import operators as ops
from upsnet_b200._lib import lib

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=20)
args = ap.parse_args()
dev = torch.device("cuda", 0)
torch.manual_seed(0)

# name, N, Cin, Cout, H, W, k, residual (None / "res" / "up2"), pair_group
LAYERS = [
    ("fpn/rpn 3x3 256->256 @256x512", 1, 256, 256, 256, 512, 3, None, 0),
    ("fpn/rpn 3x3 256->256 @128x256", 1, 256, 256, 128, 256, 3, None, 0),
    ("mask head 3x3 256->256 256 rois 14x14", 256, 256, 256, 14, 14, 3, None, 0),
    ("res2 conv2 3x3 64->64 @256x512", 1, 64, 64, 256, 512, 3, None, 0),
    ("res3 conv2 3x3 128->128 @128x256", 1, 128, 128, 128, 256, 3, None, 0),
    ("res4 conv2 3x3 256->256 @64x128", 1, 256, 256, 64, 128, 3, None, 0),
    ("res5 conv2 3x3 512->512 @32x64", 1, 512, 512, 32, 64, 3, None, 0),
    ("res2 conv3 1x1 64->256 +res @256x512", 1, 64, 256, 256, 512, 1, "res", 0),
    ("res3 conv3 1x1 128->512 +res @128x256", 1, 128, 512, 128, 256, 1, "res", 0),
    ("res4 conv3 1x1 256->1024 +res @64x128", 1, 256, 1024, 64, 128, 1, "res", 0),
    ("fpn lateral 1x1 512->256 +up2 @128x256", 1, 512, 256, 128, 256, 1, "up2", 0),
    ("fc6 1x1 12544->1024 1000 rois", 1000, 12544, 1024, 1, 1, 1, None, 0),
    ("mask deconv as 1x1 256->4x256 256 rois 14x14", 256, 256, 1024, 14, 14, 1, None, 256),
]


def gpu_ms(fn):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / args.reps


def make(mode, N, Cin, Cout, H, W, k, res, pg):
    x = torch.randn(N, Cin, H, W, device=dev)
    w = torch.randn(Cout, Cin, k, k, device=dev) / (Cin * k * k) ** 0.5
    b = torch.randn(Cout, device=dev)
    r = None
    if res == "res":
        r = torch.randn(N, Cout, H, W, device=dev)
    elif res == "up2":
        r = torch.randn(N, Cout, H // 2, W // 2, device=dev)
    if mode == "bf16":
        def cl(t):
            return t.bfloat16().contiguous(memory_format=torch.channels_last)
        x = cl(x)
        r = None if r is None else cl(r)
        kw = dict(precision=2, out_format="nhwc", out_dtype=torch.bfloat16)
    else:
        x = ops.Pair.from_float(x)
        r = None if r is None else ops.Pair.from_float(r)
        kw = dict(precision=1)
    if pg:
        kw["pair_group"] = pg
    return lambda: U.conv2d(x, w, b, 1, k // 2, 1, residual=r, residual_up2=res == "up2", relu=True, **kw)


print("H100 / power limit and clocks: see nvidia-smi --query-gpu=name,power.limit,clocks.sm --format=csv")
print("%-46s %-12s %9s %9s %9s" % ("layer", "mode", "ms", "TFLOP/s", "exec TF/s"))
for name, N, Cin, Cout, H, W, k, res, pg in LAYERS:
    flops = 2.0 * N * H * W * Cout * Cin * k * k
    modes = [("bf16", 0)] if not pg else []
    modes += [("pair", 64), ("pair", 128)]
    for mode, bn in modes:
        if mode == "bf16" and res == "up2":
            continue
        U.set_precision("bf16" if mode == "bf16" else "bf16x3")
        assert lib().upsnet_tma_set_tile_n(bn) == 0
        try:
            ms = gpu_ms(make(mode, N, Cin, Cout, H, W, k, res, pg))
        finally:
            lib().upsnet_tma_set_tile_n(0)
        passes = 3 if mode == "pair" else 1
        label = mode + (" N=%d" % bn if bn else "")
        print("%-46s %-12s %9.4f %9.1f %9.1f" % (name, label, ms, flops / ms / 1e9, passes * flops / ms / 1e9), flush=True)
U.set_precision("fp32")
