"""The arithmetic of the dense-conv backward kernels (csrc/conv_backward.cu) restated in torch, and its error bounds.

* apriori(prec, grad, K, splits): the constant c of |kernel - fp64| <= c * (sum of |terms|) + 1e-6 derived in
  tests/test_gpu_conv_backward.py, for a gradient element made of K products.
* dgrad / wgrad: the kernels' formulation at tiny sizes, evaluated in float64 on the operands the kernels see (hi/lo
  pairs, or bf16): dX = conv(g, W') with W'[ci][co] the tap-flipped transpose and padding d (k - 1) - p; dW per tap as
  the pixel sum of g times x shifted by the tap, over K splits of the flattened pixels; dgrad_stride2: the stride-2
  1x1 dX as the compact 1x1 result scattered to the even pixels.  Keyword arguments plant the faults the CPU test shows
  the bounds reject: an unflipped tap, a one-pixel shift, a dropped K split, one 64-channel tile of dX made from the
  neighbouring tile's weight rows, the N images read as one tall image (a tap past an image's last row reads the next
  image's first row), the compact stride-2 result scattered to the odd pixels or one pixel off.
"""
import math

import torch
import torch.nn.functional as F


def apriori(prec, grad, K, splits=1):
    if grad == "db":
        return 2.0 ** -23
    if grad == "dres":
        return 2.0 ** -22
    if prec == "bf16x3":
        return 3 * 2.0 ** -16 + 3 * math.ceil(K / 16) * 2.0 ** -23 + splits * 2.0 ** -24
    return 2 * 2.0 ** -8 + 2.0 ** -16 + math.ceil(K / 16) * 2.0 ** -23 + splits * 2.0 ** -24


def split(v):
    """(hi, lo) of float32 values as float64: hi = bf16(v), lo = bf16(v - hi)."""
    v = v.float()
    hi = v.to(torch.bfloat16).float()
    lo = (v - hi).to(torch.bfloat16).float()
    return hi.double(), lo.double()


def _products(a, b, prec, op):
    """op summed over the products the kernel issues: lo*hi + hi*lo + hi*hi (bf16x3) or hi*hi (bf16)."""
    ah, al = split(a)
    bh, bl = split(b)
    if prec == "bf16":
        return op(ah, bh)
    return op(al, bh) + op(ah, bl) + op(ah, bh)


def dgrad(g, weight, padding, dilation, prec, flip=True, tile_from=None, stacked=False):
    """dX of a stride-1 conv from g [N,Cout,Ho,Wo] (float32, already masked).  tile_from=t: the 64 dX channels of tile
    t computed from the weight rows of tile t + 1; stacked (2 p = d (k - 1), so dX has the size of g): the N images of
    g read as one image N * Ho rows high."""
    kh, kw = weight.shape[2:]
    wt = weight.transpose(0, 1)
    if flip:
        wt = wt.flip(2, 3)
    if tile_from is not None:
        t = tile_from * 64
        wt = wt.clone()
        wt[t:t + 64] = wt[t + 64:t + 128]
    pad = (dilation * (kh - 1) - padding, dilation * (kw - 1) - padding)
    if not stacked:
        return _products(g, wt.contiguous(), prec, lambda a, b: F.conv2d(a, b, None, 1, pad, dilation))
    N, C, Ho, Wo = g.shape
    tall = g.transpose(0, 1).reshape(1, C, N * Ho, Wo)
    dx = _products(tall, wt.contiguous(), prec, lambda a, b: F.conv2d(a, b, None, 1, pad, dilation))
    return dx.reshape(dx.shape[1], N, -1, dx.shape[3]).transpose(0, 1)


def dgrad_stride2(g, weight, H, W, prec, scatter="even"):
    """dX [N,Cin,H,W] of a 1x1 / stride-2 conv from g [N,Cout,(H+1)/2,(W+1)/2]: the compact 1x1 result of g with
    W^T, placed at the even pixels (h, w) = (2i, 2j), zero elsewhere.  scatter='odd': at (2i+1, 2j+1); 'shift': at
    (2i, 2j+1); what falls outside the image is dropped."""
    wt = weight.transpose(0, 1).contiguous()
    compact = _products(g, wt, prec, lambda a, b: F.conv2d(a, b))
    N, Cin, Hc, Wc = compact.shape
    dx = torch.zeros((N, Cin, H, W), dtype=torch.float64)
    h0, w0 = {"even": (0, 0), "odd": (1, 1), "shift": (0, 1)}[scatter]
    nh, nw = len(range(h0, H, 2)), len(range(w0, W, 2))
    dx[:, :, h0::2, w0::2] = compact[:, :, :nh, :nw]
    return dx


def wgrad(x, g, kh, kw, padding, dilation, prec, splits=1, drop=None, shift=0):
    """dW [Cout,Cin,kh,kw] of a stride-1 conv: per tap, sum over the output pixels of g times x at the tap's offset (zero
    outside the image), the flattened pixels cut into `splits` contiguous ranges added in order (drop: a range left
    out; shift: x read one pixel off along W)."""
    N, Cin, H, W = x.shape
    _, Cout, Ho, Wo = g.shape
    xp = F.pad(x, (padding, padding + abs(shift), padding, padding))
    dw = torch.zeros((Cout, Cin, kh, kw), dtype=torch.float64)
    P = N * Ho * Wo
    bounds = [P * s // splits for s in range(splits + 1)]
    for ki in range(kh):
        for kj in range(kw):
            h0, w0 = ki * dilation, kj * dilation + shift
            xt = xp[:, :, h0:h0 + Ho, w0:w0 + Wo].permute(0, 2, 3, 1).reshape(P, Cin)
            gt = g.permute(0, 2, 3, 1).reshape(P, Cout)
            for s in range(splits):
                if s == drop:
                    continue
                a, b = bounds[s], bounds[s + 1]
                dw[:, :, ki, kj] += _products(gt[a:b], xt[a:b], prec, lambda u, v: u.t() @ v)
    return dw


def reference(x, weight, dy, padding, dilation, y=None, stride=1):
    """float64 autograd of F.conv2d and the sums of |terms|: (g, dx, dw, bound dx, bound dw); y: the forward output
    whose [y > 0] masks dy (ReLU), or None."""
    g = dy.double() * (y > 0).double() if y is not None else dy.double()
    xs = x.double().requires_grad_(True)
    ws = weight.double().requires_grad_(True)
    dx, dw = torch.autograd.grad(F.conv2d(xs, ws, None, stride, padding, dilation), (xs, ws), g)
    xa = x.double().abs().requires_grad_(True)
    wa = weight.double().abs().requires_grad_(True)
    bx, bw = torch.autograd.grad(F.conv2d(xa, wa, None, stride, padding, dilation), (xa, wa), g.abs())
    return g, dx, dw, bx, bw
