"""Timing / ncu driver for the window-staged deformable conv on pairs (csrc/dcn_win.cu) next to the global-gather kernel.
  python scripts/prof_dcn_win.py            -> CUDA-event timings for several offset distributions: the window kernel with
                                               N tile 128 and 32 (forced; "-" where 128 does not apply) and as chosen per
                                               launch, and the global-gather kernel; algorithmic TFLOP/s (one pass)
  ncu --set full --clock-control none --import-source on -k regex:dcn_win -s 2 -c 1 python scripts/prof_dcn_win.py ncu
"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import upsnet_b200 as U
from upsnet_b200 import operators as ops
from upsnet_b200._lib import lib
from upsnet_b200.operators import Pair
dev = torch.device("cuda", 0)
torch.manual_seed(0)
U.set_precision("bf16x3")
ops.DCN_WINDOW.update(on=True, min_pixels=0)


def act(n, c, h, w): return Pair.from_float(torch.randn(n, c, h, w, device=dev))
def wgt(co, ci, k): return torch.randn(co, ci, k, k, device=dev) / (ci * k * k) ** 0.5


def offsets(kind, h, w):
    if kind == "zero":
        return torch.zeros(1, 18, h, w, device=dev)
    if kind == "small":
        return torch.randn(1, 18, h, w, device=dev) * 0.5
    if kind == "tapbias":
        return (torch.randn(1, 18, 1, 1, device=dev) * 1.5 + torch.randn(1, 18, h, w, device=dev) * 0.5).contiguous()
    if kind == "rand1.5":
        return torch.randn(1, 18, h, w, device=dev) * 1.5
    if kind == "rand4":
        return torch.randn(1, 18, h, w, device=dev) * 4.0
    raise ValueError(kind)


def gpu_ms(fn, iters=10):
    fn(); fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


shapes = [(256, 128, 256, 512), (128, 128, 256, 512), (256, 128, 128, 256), (256, 128, 64, 128), (256, 128, 32, 64),
          (256, 256, 100, 168), (512, 512, 50, 84)]
if len(sys.argv) > 1 and sys.argv[1] == "ncu":
    x, w = act(1, 256, 256, 512), wgt(128, 256, 3)
    off = offsets(sys.argv[2] if len(sys.argv) > 2 else "tapbias", 256, 512)
    for _ in range(3):
        U.deform_conv(x, off, w, None, 1, 1, 1, relu=True)
    torch.cuda.synchronize()
    sys.exit(0)
def window_ms(bn, fn):
    assert lib().upsnet_dcn_set_tile_n(bn) == 0
    try:
        return gpu_ms(fn)
    finally:
        lib().upsnet_dcn_set_tile_n(0)


for cin, cout, h, w_ in shapes:
    x, w = act(1, cin, h, w_), wgt(cout, cin, 3)
    fl = 2.0 * h * w_ * cout * cin * 9
    for kind in ("zero", "small", "tapbias", "rand1.5", "rand4"):
        off = offsets(kind, h, w_)
        run = lambda: U.deform_conv(x, off, w, None, 1, 1, 1, relu=True)
        ops.DCN_WINDOW["on"] = True
        t = {bn: window_ms(bn, run) for bn in (128, 32, 0)}
        ops.DCN_WINDOW["on"] = False
        g = gpu_ms(run)
        ops.DCN_WINDOW["on"] = True
        wide = "  N128 %.3f ms (%4.0f TF/s)" % (t[128], fl / t[128] / 1e9) if cout % 128 == 0 else "  N128 -"
        print("Cin%d->%d @%dx%d off=%-8s%s  N32 %.3f ms (%4.0f TF/s)  auto %.3f ms   global-gather %.3f ms"
              % (cin, cout, h, w_, kind, wide, t[32], fl / t[32] / 1e9, t[0], g), flush=True)
