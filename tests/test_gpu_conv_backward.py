"""Dense-conv backward (csrc/conv_backward.cu behind upsnet_b200.training.conv2d / linear / conv_transpose2x2) against
autograd of F.conv2d / F.linear / F.conv_transpose2d in float64 on the device, element by element, each element against
its own bound through grad_oracle.check: |kernel - fp64| <= c * (sum of |terms|) + 1e-6.  The float64 reference takes
the same float32 x, W, b, residual and dY, and the ReLU mask of the kernel's own forward output (so that an output at
exactly 0 cannot decide the mask differently).  Run with -s to see the worst err / bound per family.  Own file = own
process (a trap in a tensor-core kernel poisons the CUDA context).

A-priori bounds (T = the sum of |terms| of the element: |W| |g| summed over the taps / channels for dX, |g| |x| summed
over the pixels for dW, |g| for d bias and d residual; K = the number of products of the element):

bf16x3 (g and x stored as hi/lo pairs, W split into hi/lo planes; lo*hi + hi*lo + hi*hi per product):
  * each operand's split: |v - hi - lo| <= 2^-8 |v - hi| <= 2^-16 |v|: 2 * 2^-16 per product; lo * lo dropped:
    |lo_a lo_b| <= 2^-16 |a b|.  Sum 3 * 2^-16 = 4.6e-5.
  * fp32 accumulation in wgmma: 3 K / 16 steps, each adding at most 2^-23 of the magnitudes (the tensor core aligns
    the addends by truncation); dW adds its K splits in fp32 afterwards (splits * 2^-24).  At K = 2304 (3x3, 256
    channels) 5.1e-5, so c = 9.7e-5 for dX; for dW K is the pixels of one split (16384 at fpn_p2 full size: 3.7e-4).
bf16 (g, x and W rounded to bf16, one product): 2 * 2^-8 + 2^-16 = 7.8e-3 per product, plus K / 16 * 2^-23.
d bias: exact fp32 terms summed in fp64 in a fixed order, rounded once: 2^-24 (c = 2^-23).  d residual: g itself (0), or
  ((g00 + g01) + g10) + g11 in fp32 for residual_up2: 3 * 2^-24 (c = 2^-22).

Measured on an NVIDIA H100 80GB HBM3 (SXM, power limit 700 W), worst err / bound over all cases: bf16x3 dX 1.73e-5,
dW 1.34e-5; bf16 dX 6.3e-3, dW 4.9e-3; d bias 3.4e-8, d residual 1.2e-7.  conv_grad_cases.TOL holds about 4x the
bf16x3 values.  The layer harness lives in tests/conv_grad_cases.py, the a-priori constants in
tests/conv_grad_oracle.py; tests/test_conv_grad_oracle_cpu.py shows they reject an unflipped tap, a one-pixel shift, a
dropped K split and a missing ReLU mask.  tests/test_gpu_conv_backward_wide.py runs the same harness at the channel
widths of the training forward.
"""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from conv_grad_cases import _check, _rand, _run_linear, _vjp, report, run_conv, run_deconv  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    yield torch.device("cuda", 0)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    report()


PRECS = ["bf16x3", "bf16"]

# every trainable layer family of UPSNet-50 at reduced size, ragged boxes (H, W not multiples of the pixel box)
FAMILIES = [
    # name, N, Cin, H, W, Cout, k, stride, pad, dil, bias, relu, res
    ("1x1 s1 +res relu", 2, 128, 13, 22, 256, 1, 1, 0, 1, True, True, "same"),
    ("1x1 s1 nobias", 2, 256, 11, 9, 64, 1, 1, 0, 1, False, False, None),
    ("1x1 s2 relu", 2, 256, 13, 22, 128, 1, 2, 0, 1, False, True, None),
    ("1x1 s2 downsample", 1, 128, 24, 17, 256, 1, 2, 0, 1, True, False, None),
    ("3x3 p1 relu", 1, 128, 19, 27, 128, 3, 1, 1, 1, True, True, None),
    ("3x3 d2 p2 relu", 1, 128, 17, 23, 64, 3, 1, 2, 2, True, True, None),
    ("fpn lat res_up2", 1, 256, 14, 22, 128, 1, 1, 0, 1, True, False, "up2"),
    ("fpn 3x3 p1", 1, 128, 15, 30, 128, 3, 1, 1, 1, True, False, None),
    ("rpn cls 3", 1, 256, 13, 21, 3, 1, 1, 0, 1, True, False, None),
    ("rpn bbox 12", 1, 256, 13, 21, 12, 1, 1, 0, 1, True, False, None),
    ("fcn score 19", 1, 128, 25, 26, 19, 1, 1, 0, 1, True, False, None),
    ("score 133", 1, 128, 9, 15, 133, 1, 1, 0, 1, True, False, None),
    ("mask score 9", 7, 256, 28, 28, 9, 1, 1, 0, 1, True, False, None),
    ("mask score 81", 3, 256, 28, 28, 81, 1, 1, 0, 1, True, False, None),
    ("mask conv 3x3 relu", 11, 256, 14, 14, 256, 3, 1, 1, 1, True, True, None),
]


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("fam", FAMILIES, ids=[f[0] for f in FAMILIES])
def test_layer_families(dev, prec, fam):
    name, N, Cin, H, W, Cout, k, s, p, d, bias, relu, res = fam
    run_conv(dev, name, prec, N, Cin, H, W, Cout, k, s, p, d, bias, relu, res, seed=len(name))


@pytest.mark.parametrize("prec", PRECS)
def test_dy_nhwc_and_no_dgrad(dev, prec):
    """dY in channels_last strides; an input that needs no gradient (fpn_lat2 on the detached res2) runs no dgrad."""
    run_conv(dev, "3x3 dy nhwc", prec, 2, 64, 10, 13, 64, 3, 1, 1, 1, True, True, None, seed=5, nhwc_dy=True)
    run_conv(dev, "lat2 no dx", prec, 1, 256, 12, 20, 128, 1, 1, 0, 1, True, False, None, seed=6, need_x=False)


@pytest.mark.parametrize("prec", PRECS)
def test_linear_heads(dev, prec):
    """fc6 (K = 12544), fc7 and the cls / bbox heads on one-pixel images."""
    _run_linear(dev, "fc6", prec, 40, 12544, 1024, True, 11)
    _run_linear(dev, "fc7", prec, 37, 1024, 1024, True, 12)
    _run_linear(dev, "cls 9", prec, 37, 1024, 9, False, 13)
    _run_linear(dev, "bbox 36", prec, 37, 1024, 36, False, 14)
    _run_linear(dev, "cls 81", prec, 37, 1024, 81, False, 15)
    _run_linear(dev, "bbox 324", prec, 37, 1024, 324, False, 16)


@pytest.mark.parametrize("prec", PRECS)
def test_deconv_2x2(dev, prec):
    """The mask branch's ConvTranspose2d(256, 256, 2, 2) + ReLU on 163 rois of 14 x 14."""
    run_deconv(dev, "deconv 2x2", prec, 163, 256, 256, 14, 21)


def test_fullsize(dev):
    """Full size, bf16x3: fpn_p2 (3x3 256->256 at 256x512), the res3 block-0 stride-2 1x1 (256 -> 128 at 256x512 ->
    128x256) and fc6 on 512 rois."""
    run_conv(dev, "full fpn_p2", "bf16x3", 1, 256, 256, 512, 256, 3, 1, 1, 1, True, False, None, seed=31)
    run_conv(dev, "full res3 s2", "bf16x3", 1, 256, 256, 512, 128, 1, 2, 0, 1, False, True, None, seed=32)
    _run_linear(dev, "full fc6", "bf16x3", 512, 12544, 1024, True, 33)


def test_shared_weight_accumulates(dev):
    """The RPN 3x3 head over P2..P6: one weight, five calls, the gradient is the sum."""
    from upsnet_b200 import training
    w = _rand((128, 128, 3, 3), dev, (2.0 / 1152) ** 0.5, 41).requires_grad_(True)
    b = _rand((128,), dev, 0.1, 42).requires_grad_(True)
    sizes = [(32, 48), (16, 24), (8, 12), (4, 6), (2, 3)]
    xs = [_rand((1, 128, h, ww), dev, 1.0, 43 + i) for i, (h, ww) in enumerate(sizes)]
    dys = [_rand((1, 128, h, ww), dev, 1.0, 53 + i) for i, (h, ww) in enumerate(sizes)]
    gw = torch.zeros(w.shape, dtype=torch.float64, device=dev)
    bw = torch.zeros_like(gw)
    for x, dy in zip(xs, dys):
        y = training.conv2d(x, w, b, 1, 1, 1, relu=True, precision="bf16x3")
        y.backward(dy)
        g = dy.double() * (y.detach() > 0).double()
        (_, gwi), (_, bwi) = _vjp(lambda a, ww: F.conv2d(a, ww, None, 1, 1), [x, w.detach()], g)
        gw += gwi
        bw += bwi
    _check("rpn shared x5", "bf16x3", "dw", w.grad, gw, bw, 32 * 48 + 64, 5 * 8)


@pytest.mark.parametrize("prec", PRECS)
def test_deterministic_and_graph_replay(dev, prec):
    """Two runs give the same bytes, and a CUDA-graph replay of the backward gives them again."""
    from upsnet_b200 import training, _lib
    p = _lib.PREC_BF16X3 if prec == "bf16x3" else _lib.PREC_BF16
    N, Cin, H, W, Cout = 1, 128, 37, 45, 128
    x = _rand((N, Cin, H, W), dev, 1.0, 61)
    w = _rand((Cout, Cin, 3, 3), dev, 0.05, 62)
    b = _rand((Cout,), dev, 0.1, 63)
    dy = _rand((N, Cout, H, W), dev, 1.0, 64)
    xs = training._stored_input(x, p)
    from upsnet_b200 import operators as ops
    y = ops.conv2d(training._kernel_input(xs, p), w, b, 1, 1, 1, relu=True, precision=p, out_dtype=torch.float32)
    geom = (N, Cin, H, W, (1, 1), (1, 1), (1, 1))

    def step():
        return training.conv2d_backward(dy, xs, y.permute(0, 2, 3, 1), w, geom, p, relu=True, has_bias=True)[:3]

    a = [t.clone() for t in step()]
    bb = [t.clone() for t in step()]
    for u, v in zip(a, bb):
        assert torch.equal(u, v)
    step()                                        # packed weights cached, allocator warm
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            out = step()
    graph.replay()
    torch.cuda.synchronize()
    for u, v in zip(a, out):
        assert torch.equal(u, v)


@pytest.mark.parametrize("prec", PRECS)
def test_forward_bytes_equal_ops(dev, prec):
    """The forward is ops.conv2d of the stored copy of x with a float32 output, byte for byte."""
    from upsnet_b200 import training, _lib, operators as ops
    p = _lib.PREC_BF16X3 if prec == "bf16x3" else _lib.PREC_BF16
    x = _rand((2, 128, 19, 23), dev, 1.0, 71)
    w = _rand((64, 128, 3, 3), dev, 0.05, 72)
    b = _rand((64,), dev, 0.1, 73)
    r = _rand((2, 64, 19, 23), dev, 1.0, 74)
    y = training.conv2d(x, w, b, 1, 1, 1, residual=r, relu=True, precision=prec)
    y_ops = ops.conv2d(training._kernel_input(training._stored_input(x, p), p), w, b, 1, 1, 1, residual=r, relu=True,
                       precision=p, out_dtype=torch.float32)
    assert torch.equal(y, y_ops)
    if prec == "bf16x3":
        s = training._stored_input(x, p)
        assert s.numel() * s.element_size() == x.numel() * x.element_size()     # the pair: the bytes of the fp32 x
        assert float(((ops.Pair(s).float() - x).abs() / x.abs().clamp_min(1e-30)).max()) <= 2.0 ** -16


def test_unsupported_raise(dev):
    from upsnet_b200 import training, _lib
    x = _rand((1, 128, 16, 16), dev)
    with pytest.raises(_lib.UpsnetError):
        training.conv2d(x, _rand((64, 128, 3, 3), dev), stride=2, padding=1)        # stride 2 with k > 1
    with pytest.raises(_lib.UpsnetError):
        training.conv2d(_rand((1, 96, 16, 16), dev), _rand((64, 96, 1, 1), dev))    # Cin % 64
    with pytest.raises(_lib.UpsnetError):
        training.conv2d(x, _rand((64, 64, 3, 3), dev), padding=1)                   # groups 2
    with pytest.raises(_lib.UpsnetError):
        training.conv_transpose2x2(x, _rand((128, 64, 3, 3), dev))                  # kernel 3
    with pytest.raises(ValueError):
        training.conv2d(x, _rand((64, 128, 1, 1), dev), precision="fp32")
