"""The layer harness of the dense-conv backward tests (tests/test_gpu_conv_backward.py, test_gpu_conv_backward_wide.py):
one layer through upsnet_b200.training.conv2d / linear / conv_transpose2x2, forward and backward, against float64
autograd of F.conv2d / F.linear / F.conv_transpose2d on the device, element by element through grad_oracle.check at the
a-priori constants of conv_grad_oracle.apriori (or TOL where it is tighter), and the forward output y against
conv_grad_oracle.forward at conv_grad_oracle.forward_c.  The float64 reference takes the same
float32 x, W, b, residual and dY, and the ReLU mask of the kernel's own forward output (so that an output at exactly 0
cannot decide the mask differently).  WORST collects the worst err / bound per (case, precision, gradient)."""
import math
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import grad_oracle as G  # noqa: E402
from conv_grad_oracle import apriori, forward, forward_c  # noqa: E402

WORST = {}
# About 4x the worst err / bound measured on the H100 (bf16x3: dX 1.73e-5 at the RPN cls head, dW 1.34e-5 at fc6), used
# where it is below the a-priori constant.  bf16: the operands' own rounding is the error (measured dX 6.3e-3, dW 4.9e-3
# against 7.8e-3 a priori), so the a-priori constant is the tolerance.  d bias (3.4e-8) and d residual (1.2e-7) are
# checked at their a-priori 1.2e-7 and 2.4e-7.
TOL = {("bf16x3", "dx"): 7e-5, ("bf16x3", "dw"): 5.5e-5}


def report(title="conv backward worst err/bound"):
    for k in sorted(WORST):
        print("%s %-40s %.3e" % (title, k, WORST[k]))


def _check(name, prec, grad, got, want, bound, K, splits=1):
    c = apriori(prec, grad, K, splits)
    tol = TOL.get((prec, grad))
    c_use = min(c, tol) if tol is not None else c
    ok, ratio = G.check(got, want, bound, c_use)
    key = "%s %s %s" % (name, prec, grad)
    WORST[key] = max(WORST.get(key, 0.0), ratio)
    assert ok, "%s: worst err/bound %.3e > c %.3e" % (key, ratio, c_use)


def _check_y(name, prec, y, x, w, b=None, stride=1, pad=0, dil=1, r=None, up2=False, relu=False):
    """The forward output y (float32 [N, Cout, Ho, Wo]) element by element against conv_grad_oracle.forward on the copy
    of x the kernel reads (the hi / lo pair of x for bf16x3, bf16(x) for bf16)."""
    from upsnet_b200 import operators as ops
    x = x.detach()
    if prec == "bf16x3":
        C, st = x.shape[1], ops.Pair.from_float(x).store
        xr = tuple(st[..., i * C:(i + 1) * C].double().permute(0, 3, 1, 2) for i in (0, 1))
    else:
        xr = x.bfloat16().double()
    want, bound, _ = forward(xr, w.detach(), None if b is None else b.detach(), stride, pad, dil,
                             None if r is None else r.detach(), up2, relu, prec)
    c = forward_c(prec, w.shape[1] * w.shape[2] * w.shape[3], int(b is not None) + int(r is not None))
    ok, ratio = G.check(y.detach(), want, bound, c)
    key = "%s %s y" % (name, prec)
    WORST[key] = max(WORST.get(key, 0.0), ratio)
    assert ok, "%s: worst err/bound %.3e > c %.3e" % (key, ratio, c)


def _rand(shape, dev, scale=1.0, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randn(shape, generator=g, device=dev) * scale


def _vjp(f, inputs, cot):
    """float64 autograd of f at `inputs` with cotangent cot, and of f at |inputs| with |cot| (the sums of |terms|)."""
    xs = [t.double().detach().requires_grad_(True) for t in inputs]
    out = f(*xs)
    grads = torch.autograd.grad(out, xs, cot.double())
    xa = [t.double().abs().detach().requires_grad_(True) for t in inputs]
    outa = f(*xa)
    bounds = torch.autograd.grad(outa, xa, cot.double().abs())
    return grads, bounds


def wgrad_splits(prec, N, Cin, H, W, Cout, k, stride=1, pad=0, dil=1):
    """The K splits of the wgrad kernel for this layer, read back from the size of its workspace."""
    from upsnet_b200 import _lib
    nb = _lib.query_bytes("conv_wgrad_workspace_bytes", N, H, W, Cin, Cout, k, k, stride, stride, pad, pad, dil, dil,
                          _lib.PREC_BF16X3 if prec == "bf16x3" else _lib.PREC_BF16)
    return max(1, nb // (4 * k * k * ((Cout + 127) // 128 * 128) * ((Cin + 127) // 128 * 128)))


def run_conv(dev, name, prec, N, Cin, H, W, Cout, k, stride=1, pad=0, dil=1, bias=True, relu=False, res=None,
             seed=0, nhwc_dy=False, need_x=True):
    """One layer: training.conv2d forward + backward vs float64 autograd.  res: None, 'same' or 'up2'."""
    from upsnet_b200 import training
    x = _rand((N, Cin, H, W), dev, 1.0, seed)
    w = _rand((Cout, Cin, k, k), dev, (2.0 / (Cin * k * k)) ** 0.5, seed + 1).requires_grad_(True)
    b = _rand((Cout,), dev, 0.1, seed + 2).requires_grad_(True) if bias else None
    Ho = (H + 2 * pad - dil * (k - 1) - 1) // stride + 1
    Wo = (W + 2 * pad - dil * (k - 1) - 1) // stride + 1
    r = None
    if res == "same":
        r = _rand((N, Cout, Ho, Wo), dev, 1.0, seed + 3).requires_grad_(True)
    elif res == "up2":
        r = _rand((N, Cout, Ho // 2, Wo // 2), dev, 1.0, seed + 3).requires_grad_(True)
    xg = x.clone().requires_grad_(need_x)
    y = training.conv2d(xg, w, b, stride, pad, dil, residual=r, residual_up2=(res == "up2"), relu=relu, precision=prec)
    assert y.shape == (N, Cout, Ho, Wo) and y.dtype == torch.float32
    _check_y(name, prec, y, x, w, b, stride, pad, dil, r, res == "up2", relu)
    dy = _rand((N, Cout, Ho, Wo), dev, 1.0, seed + 4)
    if nhwc_dy:
        dy = dy.contiguous(memory_format=torch.channels_last)
    y.backward(dy)
    g = dy.double() * (y.detach() > 0).double() if relu else dy.double()
    conv = lambda a, bw: F.conv2d(a, bw, None, stride, pad, dil)   # noqa: E731
    (gx, gw), (bx, bw) = _vjp(conv, [x, w.detach()], g)
    if need_x:
        assert xg.grad.shape == x.shape
        _check(name, prec, "dx", xg.grad, gx, bx, ((Cout + 63) // 64 * 64) * k * k)
    else:
        assert xg.grad is None
    S = wgrad_splits(prec, N, Cin, H, W, Cout, k, stride, pad, dil)
    _check(name, prec, "dw", w.grad, gw, bw, math.ceil(N * Ho * Wo / S / 64) * 64 + 64, S)
    if bias:
        _check(name, prec, "db", b.grad, g.sum((0, 2, 3)), g.abs().sum((0, 2, 3)), N * Ho * Wo)
    if res == "same":
        _check(name, prec, "dres", r.grad, g, g.abs(), 1)
    elif res == "up2":
        _check(name, prec, "dres", r.grad, F.avg_pool2d(g, 2) * 4, F.avg_pool2d(g.abs(), 2) * 4, 4)
    return y


def _run_linear(dev, name, prec, R, K, Cout, relu, seed, bias=True):
    from upsnet_b200 import training
    x = _rand((R, K), dev, 1.0, seed).requires_grad_(True)
    w = _rand((Cout, K), dev, (2.0 / K) ** 0.5, seed + 1).requires_grad_(True)
    b = _rand((Cout,), dev, 0.1, seed + 2).requires_grad_(True) if bias else None
    y = training.linear(x, w, b, relu=relu, precision=prec)
    _check_y(name, prec, y.reshape(R, Cout, 1, 1), x.reshape(R, K, 1, 1), w.reshape(Cout, K, 1, 1), b, relu=relu)
    dy = _rand((R, Cout), dev, 1.0, seed + 3)
    y.backward(dy)
    g = dy.double() * (y.detach() > 0).double() if relu else dy.double()
    (gx, gw), (bx, bw) = _vjp(lambda a, ww: F.linear(a, ww), [x.detach(), w.detach()], g)
    _check(name, prec, "dx", x.grad, gx, bx, (Cout + 63) // 64 * 64)
    _check(name, prec, "dw", w.grad, gw, bw, math.ceil(R / 64) * 64 + 64)
    if bias:
        _check(name, prec, "db", b.grad, g.sum(0), g.abs().sum(0), R)


def run_deconv(dev, name, prec, R, Cin, C, H, seed):
    """ConvTranspose2d(Cin, C, 2, 2) + ReLU on R images of H x H."""
    from upsnet_b200 import training
    x = _rand((R, Cin, H, H), dev, 1.0, seed).requires_grad_(True)
    w = _rand((Cin, C, 2, 2), dev, (2.0 / Cin) ** 0.5, seed + 1).requires_grad_(True)
    b = _rand((C,), dev, 0.1, seed + 2).requires_grad_(True)
    y = training.conv_transpose2x2(x, w, b, relu=True, precision=prec)
    assert y.shape == (R, C, 2 * H, 2 * H)
    # the 1x1 conv to 4 C channels ordered (a, b, c) the kernel runs, then the pixel shuffle
    w1 = w.detach().permute(2, 3, 1, 0).reshape(4 * C, Cin, 1, 1)
    y1 = y.detach().reshape(R, C, H, 2, H, 2).permute(0, 3, 5, 1, 2, 4).reshape(R, 4 * C, H, H)
    _check_y(name, prec, y1, x, w1, b.detach().repeat(4), relu=True)
    dy = _rand(y.shape, dev, 1.0, seed + 3)
    y.backward(dy)
    g = dy.double() * (y.detach() > 0).double()
    (gx, gw), (bx, bw) = _vjp(lambda a, ww: F.conv_transpose2d(a, ww, None, stride=2), [x.detach(), w.detach()], g)
    _check(name, prec, "dx", x.grad, gx, bx, 4 * C)
    _check(name, prec, "dw", w.grad, gw, bw, math.ceil(R * H * H / 64) * 64 + 64, 64)
    _check(name, prec, "db", b.grad, g.sum((0, 2, 3)), g.abs().sum((0, 2, 3)), R * 4 * H * H)
