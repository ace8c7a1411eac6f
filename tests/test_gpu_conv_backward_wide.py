"""Dense-conv backward at the channel widths the training forward runs, element by element against float64 autograd
(the harness of tests/conv_grad_cases.py, the bounds of tests/conv_grad_oracle.apriori), and the deformable layers at
theirs (the bounds of tests/grad_oracle.py).  Run with -s to see the worst err / bound per case.  Own file = own
process (a trap in a tensor-core kernel poisons the CUDA context).

Width decides the kernel.  dX is a forward conv of g with a float32 NHWC output, and the TMA kernel's direct-store
epilogue takes at most 256 output channels, so the dX of every layer whose forward Cin is above 256 runs on the gather
kernel (igemm_tc_kernel) with pair / bf16 input and fp32 NHWC output, a mode the inference engine never uses.

* LAYERS: one row per distinct dense signature (kind, Cin, Cout, k, stride, pad, dil, bias, relu, residual, needs dX)
  the training forward of cityscapes_r50, coco_r50 and coco_r101_dcn runs, each at a ragged reduced size (H, W not
  multiples of the 16 x 8 / 128-pixel tiles; odd H for the stride-2 rows) in both precisions; test_routes asserts the
  route each row's backward takes from the kernels it launched, all rows in one profiler session per precision.
  test_census runs the training forward of each configuration with recorders on training.conv2d / conv_transpose2x2
  and on DeformConvFunction.apply / OffsetConvFunction.apply, and fails, naming the signature, when the model calls a
  layer neither LAYERS nor DCN_LAYERS / OFFSET_CONVS covers.
* Two images in one call (N = 2) on the gather route, sized so that a 128-pixel tile straddles them.
* Full-size rows in bf16x3 at the map sizes of 1024x2048 and 800x1344, where the K-split and tile counts are training's.
* DeformConvFunction at 128..512 channels, and the deformable Bottleneck.forward_train with its offset conv.

Measured on an NVIDIA H100 80GB HBM3 (SXM, power limit 700 W), worst err / bound (all but the census take about
30 s; the census adds one child process per configuration):
  gather route (forward Cin > 256, the N = 2 and full-size rows included): bf16x3 dX 1.25e-5 (cls 9), dW 2.6e-5
  (fpn_gap: one row, so each dW element is one product); bf16 dX 4.5e-3, dW 7.5e-3 (fpn_gap);
  TMA route: bf16x3 dX 2.0e-5 (rpn cls), dW 5.4e-6; bf16 dX 6.6e-3, dW 2.5e-3;
  d bias 3.6e-8, d residual 1.3e-7 (same and up2); full-size rows bf16x3 dX <= 3.7e-6, dW <= 2.0e-6;
  DeformConvFunction y 2.9e-7, dx 1.5e-7, d offset 1.2e-8, d weight 3.2e-7, d bias 3.9e-8; the deformable
  Bottleneck's offset conv d weight 1.1e-8, d bias 3.7e-10.
The tolerances stay those of tests/test_gpu_conv_backward.py (conv_grad_cases.TOL: bf16x3 dX 7e-5, dW 5.5e-5, else the
a-priori constant; grad_oracle.TOL for the deformable layers): 4x the values above would be looser than TOL for
bf16x3, and the bf16 values are the operands' own rounding, which only the a-priori constant bounds.
"""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import conv_grad_cases as CC  # noqa: E402
import grad_oracle as G  # noqa: E402
from kernel_trace import launched_kernels_each  # noqa: E402

pytestmark = pytest.mark.gpu
PRECS = ["bf16x3", "bf16"]
ROUTE_KERNELS = ("igemm_tc_kernel", "igemm_tma_kernel", "dgrad_scatter2_kernel", "wgrad_kernel", "wgrad_reduce_kernel")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    yield torch.device("cuda", 0)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    CC.report("wide conv backward worst err/bound")


def _sig(kind, cin, cout, k=1, s=1, p=0, d=1, bias=True, relu=False, res=None, dx=True):
    return (kind, cin, cout, k, s, p, d, bias, relu, res, dx)


# name, signature, reduced size (N, H, W; linear: R rows)
LAYERS = [
    # backbone res3 - res5 (res2 is frozen: res3 block 0 reads a tensor without gradient)
    ("res3.0 conv1 s2", _sig("conv", 256, 128, s=2, relu=True, dx=False), (1, 15, 22)),
    ("res3.0 downsample", _sig("conv", 256, 512, s=2, dx=False), (1, 15, 22)),
    ("res3 conv2 3x3", _sig("conv", 128, 128, 3, 1, 1, relu=True), (1, 13, 22)),
    ("res3 conv3 +res", _sig("conv", 128, 512, relu=True, res="same"), (1, 13, 22)),
    ("res3.1 conv1", _sig("conv", 512, 128, relu=True), (1, 13, 22)),
    ("res4.0 conv1 s2", _sig("conv", 512, 256, s=2, relu=True), (1, 15, 22)),
    ("res4.0 downsample", _sig("conv", 512, 1024, s=2), (1, 15, 22)),
    ("res4 conv2 3x3", _sig("conv", 256, 256, 3, 1, 1, relu=True), (1, 11, 19)),
    ("res4 conv3 +res", _sig("conv", 256, 1024, relu=True, res="same"), (1, 11, 19)),
    ("res4.1 conv1", _sig("conv", 1024, 256, relu=True), (1, 11, 19)),
    ("res5.0 conv1 s2", _sig("conv", 1024, 512, s=2, relu=True), (1, 13, 18)),
    ("res5.0 downsample", _sig("conv", 1024, 2048, s=2), (1, 13, 18)),
    ("res5 conv2 3x3", _sig("conv", 512, 512, 3, 1, 1, relu=True), (1, 9, 13)),
    ("res5 conv3 +res", _sig("conv", 512, 2048, relu=True, res="same"), (1, 9, 13)),
    ("res5.1 conv1", _sig("conv", 2048, 512, relu=True), (1, 9, 13)),
    # FPN
    ("fpn_p5_1x1", _sig("conv", 2048, 256), (1, 9, 13)),
    ("fpn_p4_1x1 +up2", _sig("conv", 1024, 256, res="up2"), (1, 14, 22)),
    ("fpn_p3_1x1 +up2", _sig("conv", 512, 256, res="up2"), (1, 14, 22)),
    ("fpn_p2_1x1 +up2", _sig("conv", 256, 256, res="up2", dx=False), (1, 14, 22)),
    ("fpn 3x3", _sig("conv", 256, 256, 3, 1, 1), (1, 13, 22)),
    ("fpn_gap", _sig("linear", 2048, 256), (1,)),
    # RPN (its 3x3 + ReLU has the mask branch's signature)
    ("rpn / mask 3x3", _sig("conv", 256, 256, 3, 1, 1, relu=True), (3, 14, 14)),
    ("rpn cls", _sig("conv", 256, 3), (1, 13, 21)),
    ("rpn bbox", _sig("conv", 256, 12), (1, 13, 21)),
    # RCNN
    ("fc6", _sig("linear", 12544, 1024, relu=True), (37,)),
    ("fc7", _sig("linear", 1024, 1024, relu=True), (37,)),
    ("cls 9", _sig("linear", 1024, 9), (37,)),
    ("bbox 36", _sig("linear", 1024, 36), (37,)),
    ("cls 81", _sig("linear", 1024, 81), (37,)),
    ("bbox 324", _sig("linear", 1024, 324), (37,)),
    # mask branch
    ("mask deconv", _sig("deconv", 256, 256, 2, 2, relu=True), (13, 14, 14)),
    ("mask score 9", _sig("conv", 256, 9), (5, 28, 28)),
    ("mask score 81", _sig("conv", 256, 81), (3, 28, 28)),
    # semantic head: each level's 128-channel slice of the 1x1 score conv, the bias on P2's only
    ("fcn score 19", _sig("conv", 128, 19), (1, 25, 26)),
    ("fcn score 19 nobias", _sig("conv", 128, 19, bias=False), (1, 13, 13)),
    ("fcn score 133", _sig("conv", 128, 133), (1, 25, 26)),
    ("fcn score 133 nobias", _sig("conv", 128, 133, bias=False), (1, 13, 13)),
]

# deformable 3x3 (stride 1, pad 1, dil 1, bias): backbone res3 - res5 of coco_r101_dcn, the semantic head's layers
DCN_LAYERS = [
    ("res3 dcn", 128, 128, (1, 13, 22)),
    ("res4 dcn / fcn 256", 256, 256, (1, 11, 19)),
    ("res5 dcn", 512, 512, (1, 9, 13)),
    ("fcn dcn 256->128", 256, 128, (1, 13, 21)),
    ("fcn dcn 128", 128, 128, (2, 9, 15)),
]
# the offset convs in front of them (Cin -> 18, 3x3 pad 1): their gradients are checked by test_deformable_bottleneck
OFFSET_CONVS = {128, 256, 512}


def _route(sig):
    """The kernels the row's backward must launch: dX on the gather kernel when the forward Cin is above 256 (the
    direct-store epilogue's limit), on the TMA kernel otherwise, and the scatter for stride 2; dW on wgrad + reduce."""
    kind, cin, _, _, s, _, _, _, _, _, dx = sig
    want = {"wgrad_kernel", "wgrad_reduce_kernel"}
    if dx:
        want.add("igemm_tc_kernel" if cin > 256 else "igemm_tma_kernel")
        if s == 2 and kind == "conv":
            want.add("dgrad_scatter2_kernel")
    return want


def run_row(dev, name, sig, size, prec, seed):
    kind, cin, cout, k, s, p, d, bias, relu, res, dx = sig
    if kind == "linear":
        assert dx
        CC._run_linear(dev, name, prec, size[0], cin, cout, relu, seed, bias=bias)
    elif kind == "deconv":
        assert bias and relu and dx
        CC.run_deconv(dev, name, prec, size[0], cin, cout, size[1], seed)
    else:
        N, H, W = size
        CC.run_conv(dev, name, prec, N, cin, H, W, cout, k, s, p, d, bias, relu, res, seed=seed, need_x=dx)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("row", LAYERS, ids=[r[0] for r in LAYERS])
def test_layer(dev, prec, row):
    name, sig, size = row
    if sig[0] == "conv" and sig[4] == 2:
        assert size[1] % 2 == 1, "stride-2 rows run at an odd H"
    run_row(dev, name, sig, size, prec, seed=7 * LAYERS.index(row) + 3)


# N = 2 on the gather route, H W = 143 pixels per image: the second 128-pixel tile holds the end of image 0 and the
# start of image 1
TWO_IMAGES = [
    ("n2 3x3 512", _sig("conv", 512, 512, 3, 1, 1, relu=True), (2, 11, 13)),
    ("n2 1x1 1024->256", _sig("conv", 1024, 256, relu=True), (2, 11, 13)),
]


@pytest.mark.parametrize("prec", PRECS)
def test_two_images_share_a_tile(dev, prec):
    """The 3x3's taps past the last row of image 0 must read zero, not image 1's first row, and the 1x1's pixels of
    both images in one tile must each come from their own image."""
    for name, sig, size in TWO_IMAGES:
        assert _route(sig) == {"igemm_tc_kernel", "wgrad_kernel", "wgrad_reduce_kernel"}
        run_row(dev, name, sig, size, prec, seed=len(name))


def _backward_of(dev, sig, size, prec, seed):
    """The row's layer run forward on random data; -> a call of its backward that can be repeated (retain_graph)."""
    from upsnet_b200 import training
    kind, cin, cout, k, s, p, d, bias, relu, res, dx = sig
    b = CC._rand((cout,), dev, 0.1, seed + 2).requires_grad_(True) if bias else None
    if kind == "linear":
        x = CC._rand((size[0], cin), dev, 1.0, seed).requires_grad_(dx)
        w = CC._rand((cout, cin), dev, (2.0 / cin) ** 0.5, seed + 1).requires_grad_(True)
        y = training.linear(x, w, b, relu=relu, precision=prec)
    elif kind == "deconv":
        x = CC._rand((size[0], cin, size[1], size[1]), dev, 1.0, seed).requires_grad_(dx)
        w = CC._rand((cin, cout, 2, 2), dev, (2.0 / cin) ** 0.5, seed + 1).requires_grad_(True)
        y = training.conv_transpose2x2(x, w, b, relu=relu, precision=prec)
    else:
        N, H, W = size
        Ho, Wo = (H + 2 * p - d * (k - 1) - 1) // s + 1, (W + 2 * p - d * (k - 1) - 1) // s + 1
        r = None
        if res is not None:
            r = CC._rand((N, cout) + ((Ho // 2, Wo // 2) if res == "up2" else (Ho, Wo)), dev, 1.0, seed + 3)
            r.requires_grad_(True)
        x = CC._rand((N, cin, H, W), dev, 1.0, seed).requires_grad_(dx)
        w = CC._rand((cout, cin, k, k), dev, (2.0 / (cin * k * k)) ** 0.5, seed + 1).requires_grad_(True)
        y = training.conv2d(x, w, b, s, p, d, residual=r, residual_up2=res == "up2", relu=relu, precision=prec)
    dy = CC._rand(y.shape, dev, 1.0, seed + 4)
    return lambda: y.backward(dy, retain_graph=True)


@pytest.mark.parametrize("prec", PRECS)
def test_routes(dev, prec):
    """Each row's backward launches the kernels _route names, read from one profiler session for all rows (each session
    of a long process makes later ones lose their records more often).  A dispatch change fails here naming the rows
    that moved to the other route."""
    rows = LAYERS + TWO_IMAGES
    calls = [_backward_of(dev, sig, size, prec, seed=i) for i, (_, sig, size) in enumerate(rows)]
    got = launched_kernels_each(calls, lambda n: any(k in n for k in ROUTE_KERNELS))
    moved = []
    for (name, sig, _), names in zip(rows, got):
        short = {k for n in names for k in ROUTE_KERNELS if k in n}
        if short != _route(sig):
            moved.append("%s: launched %s, the table says %s" % (name, sorted(short), sorted(_route(sig))))
    assert not moved, moved


FULL = [
    # 1024 x 2048: res4.0 conv1 on res3 (128 x 256), res5.0 downsample on res4 (64 x 128), res5 3x3 at 32 x 64
    ("full res4.0 conv1 s2", (1, 512, 128, 256, 256, 1, 2, 0, 1, True, True, None)),
    ("full res5.0 downsample", (1, 1024, 64, 128, 2048, 1, 2, 0, 1, True, False, None)),
    ("full res5 3x3", (1, 512, 32, 64, 512, 3, 1, 1, 1, True, True, None)),
    # 800 x 1344: res5 at 25 x 42
    ("full coco res5 3x3", (1, 512, 25, 42, 512, 3, 1, 1, 1, True, True, None)),
    ("full coco fpn_p5_1x1", (1, 2048, 25, 42, 256, 1, 1, 0, 1, True, False, None)),
]


@pytest.mark.parametrize("row", FULL, ids=[r[0] for r in FULL])
def test_fullsize(dev, row):
    name, args = row
    CC.run_conv(dev, name, "bf16x3", *args, seed=len(name))


# ------------------------------------------------------------------------------------------------
# deformable layers at real widths
# ------------------------------------------------------------------------------------------------
def _dcn_check(family, name, got, want, bound):
    assert got is not None, (family, name, "no gradient")
    ok, ratio = G.check(got, want, bound, G.TOL[family])
    key = "%s %s" % (name, family)
    CC.WORST[key] = max(CC.WORST.get(key, 0.0), ratio)
    assert ok, "%s: worst err/bound %.3e > c %.0e" % (key, ratio, G.TOL[family])


@pytest.mark.parametrize("row", DCN_LAYERS, ids=[r[0] for r in DCN_LAYERS])
def test_deform_conv_wide(dev, row):
    """DeformConvFunction (v1, the model's op) with offsets on and around the corner and border cases
    (grad_oracle.special_offsets), as test_gpu_backward.test_deform_conv_function_vs_fp64 checks it at Cout <= 32."""
    from upsnet_b200.training import DeformConvFunction
    name, cin, cout, (N, H, W) = row
    seed = DCN_LAYERS.index(row)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, cin, H, W, generator=g).to(dev)
    off = G.special_offsets(N, 3, 3, H, W, H, W, 1, 1, 1, seed, 0.5).to(dev)
    w = (torch.randn(cout, cin, 3, 3, generator=g) / (cin * 9) ** 0.5).to(dev)
    b = torch.randn(cout, generator=g).to(dev)
    dy = torch.randn(N, cout, H, W, generator=g).to(dev)
    ins = [t.clone().requires_grad_(True) for t in (x, off, w, b)]
    y = DeformConvFunction.apply(*ins, 1, 1, 1)
    y.backward(dy)
    ref = [t.double().requires_grad_(True) for t in (x, off, w, b)]
    y64 = G.deform_conv(ref[0], ref[1], ref[2], ref[3], None, 1, 1, 1, offset32=off)
    g64 = torch.autograd.grad(y64, ref, dy.double())
    bd = G.deform_conv_bounds(x, off, w, b, None, dy, 1, 1, 1)
    _dcn_check("dcn_y", name, y, y64, bd["y"])
    for fam, key, t, r in (("dcn_dx", "x", ins[0], g64[0]), ("dcn_doffset", "offset", ins[1], g64[1]),
                           ("dcn_dweight", "weight", ins[2], g64[2]), ("dcn_dbias", "bias", ins[3], g64[3])):
        _dcn_check(fam, name, t.grad, r, bd[key])


@pytest.mark.parametrize("planes", [128, 256, 512])
def test_deformable_bottleneck(dev, monkeypatch, planes):
    """Bottleneck.forward_train with deformable=True (a res3 - res5 block of coco_r101_dcn after block 0): the DCN's
    input, offsets, folded weight and output are caught at DeformConvFunction.apply, and the gradient that reached its
    output from the device's conv3 / ReLU backward is the cotangent of a float64 restatement of the offset conv + DCN.
    d(conv1 output), the offset conv's d weight / d bias and the DCN's d weight / d bias are checked against it, the
    offset conv's with the bound propagated through it as test_gpu_backward's WithOffset test does."""
    from upsnet_b200 import training
    from upsnet_b200.model import Bottleneck
    torch.manual_seed(planes)
    blk = Bottleneck(planes * 4, planes, deformable=True).to(dev)
    oc = blk.conv2_offset
    with torch.no_grad():
        oc.weight.normal_(0, 1.0 / (planes * 9) ** 0.5)
        oc.bias.normal_(0, 1.5)
    H, W = {128: (13, 22), 256: (11, 19), 512: (9, 13)}[planes]
    x = torch.randn(1, planes * 4, H, W, device=dev, requires_grad=True)
    dy = torch.randn(1, planes * 4, H, W, device=dev)
    cap = {}
    orig = training.DeformConvFunction.apply

    def rec(data, offset, weight, bias, *rest):
        for t in (data, weight, bias):
            if t is not None and t.requires_grad:
                t.retain_grad()
        y = orig(data, offset, weight, bias, *rest)
        y.retain_grad()
        cap.update(x=data, off=offset.detach(), w=weight, b=bias, y=y, rest=rest)
        return y

    monkeypatch.setattr(training.DeformConvFunction, "apply", staticmethod(rec))
    blk.forward_train(x, "bf16x3").backward(dy)
    assert cap["rest"] == (1, 1, 1)
    xx, w2, b2, gy = cap["x"], cap["w"], cap["b"], cap["y"].grad
    with torch.enable_grad():
        xs, ow, ob, ws, bs = (t.detach().double().requires_grad_(True) for t in (xx, oc.weight, oc.bias, w2, b2))
        off = F.conv2d(xs, ow, ob, padding=1)
        off.retain_grad()
        G.deform_conv(xs, off, ws, bs, None, 1, 1, 1, offset32=cap["off"]).backward(gy.double())
    bd = G.deform_conv_bounds(xx, off.detach(), w2, b2, None, gy, 1, 1, 1)
    up = bd["offset"] + off.grad.abs()          # d(offset) is within c * bound of fp64: propagate that bound
    xa, wa = xx.detach().double().abs(), oc.weight.detach().double().abs()
    cx = torch.nn.grad.conv2d_input(xa.shape, wa, up, padding=1)
    cw = torch.nn.grad.conv2d_weight(xa, wa.shape, up, padding=1)
    name = "bottleneck %d" % planes
    _dcn_check("dcn_dx", name, xx.grad, xs.grad, bd["x"] + cx)
    _dcn_check("dcn_dweight", name + " offset conv", oc.weight.grad, ow.grad, cw)
    _dcn_check("dcn_dbias", name + " offset conv", oc.bias.grad, ob.grad, up.sum((0, 2, 3)))
    _dcn_check("dcn_dweight", name, w2.grad, ws.grad, bd["weight"])
    if b2.requires_grad:            # the folded BN shift: a constant of the step unless the BN parameters train
        _dcn_check("dcn_dbias", name, b2.grad, bs.grad, bd["bias"])


# ------------------------------------------------------------------------------------------------
# census: every layer the training forward calls is a row of the tables above
# ------------------------------------------------------------------------------------------------
def _pair1(v):
    v = tuple(v) if isinstance(v, (tuple, list)) else (v, v)
    assert v[0] == v[1], v
    return int(v[0])


def _record(monkeypatch):
    import inspect

    from upsnet_b200 import training
    seen = set()
    conv2d, deconv = training.conv2d, training.conv_transpose2x2
    dcn, offc = training.DeformConvFunction.apply, training.OffsetConvFunction.apply
    conv_sig, deconv_sig = inspect.signature(conv2d), inspect.signature(deconv)

    def conv_rec(*a, **kw):
        b = conv_sig.bind(*a, **kw)
        b.apply_defaults()
        v = b.arguments
        x, w = v["x"], v["weight"]
        N, cin, H, W = x.shape
        kind = "linear" if H == W == 1 else "conv"
        res = None if v["residual"] is None else ("up2" if v["residual_up2"] else "same")
        seen.add(_sig(kind, cin, w.shape[0], w.shape[2], _pair1(v["stride"]), _pair1(v["padding"]),
                      _pair1(v["dilation"]), v["bias"] is not None, bool(v["relu"]), res, x.requires_grad))
        return conv2d(*a, **kw)

    def deconv_rec(*a, **kw):
        b = deconv_sig.bind(*a, **kw)
        b.apply_defaults()
        v = b.arguments
        x, w = v["x"], v["weight"]
        seen.add(_sig("deconv", x.shape[1], w.shape[1], w.shape[2], _pair1(v["stride"]), 0, 1, v["bias"] is not None,
                      bool(v["relu"]), None, x.requires_grad))
        return deconv(*a, **kw)

    def dcn_rec(x, offset, weight, bias=None, stride=1, padding=0, dilation=1):
        seen.add(("dcn", x.shape[1], weight.shape[0], weight.shape[2], _pair1(stride), _pair1(padding),
                  _pair1(dilation), bias is not None))
        return dcn(x, offset, weight, bias, stride, padding, dilation)

    def offc_rec(x, weight, bias):
        seen.add(("offset", x.shape[1], weight.shape[0]))
        return offc(x, weight, bias)

    monkeypatch.setattr(training, "conv2d", conv_rec)
    monkeypatch.setattr(training, "conv_transpose2x2", deconv_rec)
    monkeypatch.setattr(training.DeformConvFunction, "apply", staticmethod(dcn_rec))
    monkeypatch.setattr(training.OffsetConvFunction, "apply", staticmethod(offc_rec))
    return seen


CONFIGS = {"cityscapes_r50": (256, 512, "cityscapes", 9), "coco_r50": (256, 384, "coco", 81),
           "coco_r101_dcn": (256, 384, "coco", 81)}


def _census(config, monkeypatch):
    """The layer signatures one training forward of a synthetic model of the configuration calls (depth 2, 2, 2, 2:
    block 0 and one later block per stage, which have all the signatures of the full depth)."""
    import train_forward_oracle as TF

    from upsnet_b200.model import UPSNetConfig
    from upsnet_b200.synthetic import synthetic_model
    from upsnet_b200.training import PanopticLabels, RPNTargets
    dev = torch.device("cuda", 0)
    H, W, dataset, classes = CONFIGS[config]
    m = synthetic_model(getattr(UPSNetConfig, config)(), depth=(2, 2, 2, 2), seed=1, device=dev)
    entry, lmap = TF.synthetic_entry(2, H, W, 8, num_classes=classes)
    label = {"roidb": entry}
    np.random.seed(0)
    label.update(RPNTargets(max_size=max(H, W)).from_roidb(entry, 1.0, dev))
    label.update(PanopticLabels(dataset=dataset, with_roi=dataset == "coco").from_roidb(entry, lmap, (H, W), 1.0, dev))
    data = {"data": TF.image(3, H, W).to(dev), "im_info": np.array([[H, W, 1.0]], np.float32)}
    seen = _record(monkeypatch)
    m(data, label)
    return seen


_CHILD = """
import json, sys
sys.path[:0] = [%r, %r]
import pytest
import test_gpu_conv_backward_wide as T
with pytest.MonkeyPatch.context() as mp:
    print(json.dumps(sorted(T._census(%r, mp), key=repr)))
"""


@pytest.mark.parametrize("config", list(CONFIGS))
def test_census(dev, config):
    """The census runs in a child process: after the whole training forward of a model has run in the test process,
    torch.profiler sessions of later test files lose their kernel records (tests/kernel_trace.py), so the model's
    forward is kept out of it."""
    import json
    import subprocess
    here = os.path.dirname(os.path.abspath(__file__))
    out = subprocess.run([sys.executable, "-s", "-c", _CHILD % (here, os.path.dirname(here), config)],
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    seen = {tuple(s) for s in json.loads(out.stdout.strip().splitlines()[-1])}
    dense = {r[1] for r in LAYERS}
    dcn = {("dcn", cin, cout, 3, 1, 1, 1, True) for _, cin, cout, _ in DCN_LAYERS}
    offc = {("offset", c, 18) for c in OFFSET_CONVS}
    assert any(s[0] == "conv" for s in seen) and any(s[0] == "linear" for s in seen), sorted(seen, key=repr)
    assert any(s[0] == "deconv" for s in seen), sorted(seen, key=repr)
    assert any(s[0] == "dcn" for s in seen) and any(s[0] == "offset" for s in seen), sorted(seen, key=repr)
    missing = sorted((s for s in seen - dense - dcn - offc), key=repr)
    assert not missing, "%s calls layers no test covers: %s" % (config, missing)
