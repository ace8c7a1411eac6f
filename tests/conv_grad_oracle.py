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
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import grad_oracle as G  # noqa: E402


def apriori(prec, grad, K, splits=1):
    if grad == "y":
        # forward accumulation of K exact products per output (tests/test_gpu_conv_forward_fp64.py): the tensor core adds
        # the 16 products of one wgmma step to the fp32 accumulator with at most 2 * 2^-24 of the magnitudes, three MMAs
        # per step in bf16x3; the CUDA-core kernel chains K fp32 FMAs
        if prec == "fp32":
            return K * 2.0 ** -24
        return (3 if prec == "bf16x3" else 1) * math.ceil(K / 16) * 2.0 ** -23
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


EPI = 2.0 ** -23               # one fp32 add of the epilogue (bias, residual), relative to the bound
SIGMOID_SLACK = 2.0 ** -21     # expf (2 ulp), the add and the division of 1 / (1 + e^-o), relative to the result
# About 4x the worst forward err / bound measured on an NVIDIA H100 80GB HBM3 (SXM, power limit 700 W), used where it is
# below the a-priori constant: bf16x3 3.1e-6 (fc6, K = 12544: the gather kernel on the engine's rows and the training
# forward), bf16 1.0e-6 (training forward; the engine's rows 5.4e-7), fp32 4.0e-7 (res4.0 downsample on the CUDA-core
# kernel)
FWD_TOL = {"bf16x3": 1.2e-5, "bf16": 4e-6, "fp32": 1.6e-6}


def forward_c(prec, K, adds):
    """The constant c of |kernel - forward| <= c * bound + slack + 1e-6 for an output made of K products and `adds`
    epilogue additions: the a-priori accumulation and epilogue terms, or FWD_TOL[prec] where that is tighter."""
    c = apriori(prec, "y", K) + adds * EPI
    return min(c, FWD_TOL[prec]) if prec in FWD_TOL else c


def store_slack(y, bound, c, out):
    """The rounding of the stored result o, |o| <= |y| + c * bound: half a bf16 ulp of |o| (bf16 output), the hi / lo
    split's 2^-17 |o| (pair output), nothing (fp32)."""
    top = y.abs() + c * bound
    if out == "bf16":
        return G.half_ulp_bf16(top)
    if out == "pair":
        return 2.0 ** -17 * top
    return torch.zeros_like(y)


def _split_rne(v, trunc=False):
    hi = G.bf16_round(v, trunc)
    return hi, G.bf16_round(v - hi, trunc)


def forward(x, weight, bias=None, stride=1, padding=0, dilation=1, residual=None, residual_up2=False, relu=False,
            prec="bf16x3", sigmoid_from=None, fault=None, dtype=torch.float64):
    """(y, bound, slack) in float64 of one dense conv as the forward kernels compute it (csrc/igemm_tma.cu,
    csrc/igemm_tc.cu, csrc/igemm_simt.cu): the exact sum of the products the kernel issues, on the operands it sees,
    then bias, residual (same size, or nearest x2 with residual_up2), ReLU and the sigmoid of the channels from
    sigmoid_from on.  bound: the sum of |terms| (products, bias, residual), over 4 on the sigmoid channels; slack: the
    sigmoid's own rounding (None without one).
      x: the activation values the kernel reads, a float tensor [N,Cin,H,W], or the tuple (hi, lo) of a pair.
      weight: fp32, split by upsnet_igemm_pack_weight into hi = bf16(w), lo = bf16(w - hi) (round to nearest even).
      prec 'bf16x3': lo*hi + hi*lo + hi*hi, fp32 activations split the same way in the kernel; 'bf16': hi*hi, fp32
      activations rounded to bf16; 'fp32': the plain products (CUDA-core kernel).  residual: the values the epilogue
      adds (hi + lo of a pair residual).
    Planted faults for tests/test_conv_grad_oracle_cpu.py: 'shift' (every tap reads one pixel to the right), 'stacked'
    (the N images read as one tall image: a tap past the last row of one image reads the next one's first row),
    'drop_kblock' (the last 64-channel k-block of the last tap left out), 'tile_from' (output channels 0..63 computed
    from the weight rows 64..127), 'drop_lohi' (the lo*hi MMA left out), 'trunc' (the activation split, or the bf16
    rounding, truncates), 'odd' (a stride-2 1x1 reads the odd pixels), 'up2_off' (the up2 residual read at column
    (w + 1) / 2), 'bias_next' (channel co gets the bias of co + 1), 'sigmoid_early' (the sigmoid starts one channel
    early), 'relu_first' (ReLU applied before the residual).
    dtype=torch.float32 sums the products (exact in fp32 but for prec 'fp32') and runs the epilogue in fp32 instead: an
    emulation of the kernels' accumulation that the bounds must accept."""
    dt = torch.float64
    Cout, _, kh, kw = weight.shape
    trunc = fault == "trunc"
    if isinstance(x, tuple):
        assert prec == "bf16x3", "pair activations belong to precision bf16x3"
        xh, xl = (t.to(dt) for t in x)
    else:
        xv = x.to(dt)
        if prec == "bf16x3":
            xh, xl = _split_rne(xv, trunc)
        elif prec == "bf16":
            xh = G.bf16_round(xv, trunc)
    w = weight.to(dt)
    if fault == "tile_from":
        w = w.clone()
        w[0:64] = w[64:128]
    if fault == "drop_kblock":
        w = w.clone()
        w[:, -64:, -1, -1] = 0
    # (activation, weight, |weight| of the products it stands for); hi*hi + hi*lo as one product with hi + lo (exact in
    # float64: 8 by 17 bits), so that a large layer needs two float64 convolutions instead of three
    if prec == "fp32":
        terms = [(xv, w, w.abs())]
    else:
        wh, wl = _split_rne(w)
        terms = [(xh, wh, wh.abs())] if prec == "bf16" else [(xh, wh + wl, wh.abs() + wl.abs())]
        if prec == "bf16x3" and fault != "drop_lohi":
            terms.append((xl, wh, wh.abs()))
    s = stride if isinstance(stride, int) else stride[0]

    def conv(a, b):
        if s != 1 and kh == kw == 1:          # the strided view of a 1x1 / pad 0 layer: every s-th row and pixel
            Ho, Wo = (a.shape[2] - 1) // s + 1, (a.shape[3] - 1) // s + 1
            o = 1 if fault == "odd" else 0
            v = torch.zeros(a.shape[:2] + (Ho, Wo), dtype=a.dtype, device=a.device)
            part = a[:, :, o::s, o::s]
            v[:, :, :part.shape[2], :part.shape[3]] = part
            a = v
        if fault == "shift":
            a = F.pad(a, (0, 1))[..., 1:]
        if fault == "stacked":
            N, C, H, W = a.shape
            tall = a.transpose(0, 1).reshape(1, C, N * H, W)
            y = F.conv2d(tall, b, None, 1, padding, dilation)
            return y.reshape(Cout, N, -1, y.shape[3]).transpose(0, 1)
        return F.conv2d(a, b, None, 1 if kh == kw == 1 else s, padding, dilation)

    def rnd(t):
        return t.to(dtype).double()

    y = rnd(sum(conv(a.to(dtype), b.to(dtype)).double() for a, b, _ in terms))
    bound = sum(conv(a.abs(), ba) for a, _, ba in terms)
    if bias is not None:
        bv = bias.to(dt)
        if fault == "bias_next":
            bv = torch.cat([bv[1:], bv[:1]])
        y = rnd(y + bv.view(1, -1, 1, 1))
        bound = bound + bv.abs().view(1, -1, 1, 1)
    if residual is not None:
        r = residual.to(dt)
        if residual_up2:
            r = r.repeat_interleave(2, 2)
            cols = torch.arange(y.shape[3], device=y.device) // 2
            if fault == "up2_off":
                cols = ((torch.arange(y.shape[3], device=y.device) + 1) // 2).clamp_max(r.shape[3] - 1)
            r = r[..., cols]
        if fault == "relu_first":
            y = y.clamp_min(0)
        y = rnd(y + r)
        bound = bound + r.abs()
    if relu and fault != "relu_first":
        y = y.clamp_min(0)
    slack = None
    if sigmoid_from is not None:
        s0 = sigmoid_from - 1 if fault == "sigmoid_early" else sigmoid_from
        y, bound = y.clone(), bound.clone()
        y[:, s0:] = rnd(torch.sigmoid(y[:, s0:]))
        bound[:, s0:] = bound[:, s0:] / 4
        slack = torch.zeros_like(y)
        slack[:, s0:] = SIGMOID_SLACK * y[:, s0:]
    return y, bound, slack


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
