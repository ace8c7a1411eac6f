"""CPU check that the bounds of tests/test_gpu_conv_backward.py have teeth: a torch restatement of the dense-conv
backward arithmetic (tests/conv_grad_oracle.py: hi/lo pairs or bf16 operands, flipped-tap dgrad, per-tap wgrad over K
splits, the stride-2 1x1 dX scattered from its compact result) passes grad_oracle.check at the a-priori constants, and
each planted fault fails it: a tap not flipped, x read one pixel off, one K split dropped, the ReLU mask missing, and
the errors a wide layer's dX route could make: one 64-channel tile of dX from the neighbouring tile's weight rows, a
3x3 tap past the last row of one image reading the next image's first row (N = 2, as when a 128-pixel tile of the
flattened pixels straddles two images), the compact stride-2 result scattered to the odd pixels or one pixel off.

The forward (conv_grad_oracle.forward, the bounds of tests/test_gpu_conv_forward_fp64.py): its sums in fp32 pass
forward_c in every precision, and each planted fault fails it.  Swept over K = Cin * k * k (powers of two, 1x1 layers, a
3x3 for the stacked images), every fault is still rejected at K = 131072 (the largest K tried; the widest layer the engine
runs is fc6, K = 12544) in every precision but one: a truncating hi / lo split of fp32 activations at bf16x3 changes
each product by about 2^-17 of its size with a random sign, and is rejected only up to K = 128.  Pair activations, the
engine's bf16x3 input, are split on the host by Pair.from_float and not in the kernel."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import conv_grad_oracle as CG  # noqa: E402
import grad_oracle as G  # noqa: E402

CASES = [(3, 1, 1), (3, 2, 2), (1, 0, 1)]      # k, padding, dilation


def _layer(k, seed):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn((2, 16, 7, 9), generator=gen)
    w = torch.randn((12, 16, k, k), generator=gen) * (2.0 / (16 * k * k)) ** 0.5
    return x, w, gen


def _run(prec, k, pad, dil, relu=True, flip=True, shift=0, drop=None, mask=True, splits=3):
    x, w, gen = _layer(k, 7 * k + pad)
    y = F.conv2d(x, w, None, 1, pad, dil)
    dy = torch.randn(y.shape, generator=gen)
    g, dx, dw, bx, bw = CG.reference(x, w, dy, pad, dil, y if relu else None)
    g_kernel = (dy * (y > 0).float()) if (relu and mask) else dy
    ex = CG.dgrad(g_kernel, w, pad, dil, prec, flip=flip)
    ew = CG.wgrad(x, g_kernel, k, k, pad, dil, prec, splits=splits, drop=drop, shift=shift)
    P = y.shape[0] * y.shape[2] * y.shape[3]
    okx, rx = G.check(ex, dx, bx, CG.apriori(prec, "dx", 12 * k * k))
    okw, rw = G.check(ew, dw, bw, CG.apriori(prec, "dw", P, splits))
    return okx, okw, rx, rw


@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
@pytest.mark.parametrize("case", CASES)
def test_restatement_passes(prec, case):
    okx, okw, rx, rw = _run(prec, *case)
    assert okx and okw, (rx, rw)


@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_tap_not_flipped_fails(prec):
    okx, _, _, _ = _run(prec, 3, 1, 1, flip=False)
    assert not okx


@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_pixel_shift_fails(prec):
    _, okw, _, _ = _run(prec, 3, 1, 1, shift=1)
    assert not okw


@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_dropped_split_fails(prec):
    _, okw, _, _ = _run(prec, 3, 2, 2, drop=1)
    assert not okw


@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_missing_relu_mask_fails(prec):
    okx, okw, _, _ = _run(prec, 3, 1, 1, mask=False)
    assert not okx and not okw


def _wide(prec, tile_from=None, stacked=False):
    """dX of a 3x3 / pad 1 conv, 192 -> 24 channels (three 64-channel dX tiles), N = 2 images of 5 x 6."""
    gen = torch.Generator().manual_seed(23)
    x = torch.randn((2, 192, 5, 6), generator=gen)
    w = torch.randn((24, 192, 3, 3), generator=gen) * (2.0 / (192 * 9)) ** 0.5
    dy = torch.randn((2, 24, 5, 6), generator=gen)
    g, dx, _, bx, _ = CG.reference(x, w, dy, 1, 1)
    ex = CG.dgrad(dy, w, 1, 1, prec, tile_from=tile_from, stacked=stacked)
    return G.check(ex, dx, bx, CG.apriori(prec, "dx", 64 * 9))


@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_wide_restatement_passes(prec):
    ok, r = _wide(prec)
    assert ok, r


@pytest.mark.parametrize("tile", [0, 1])
@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_dx_tile_from_neighbour_fails(prec, tile):
    assert not _wide(prec, tile_from=tile)[0]


@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_tap_reads_next_image_fails(prec):
    assert not _wide(prec, stacked=True)[0]


def _stride2(prec, H, W, scatter):
    gen = torch.Generator().manual_seed(H * W)
    x = torch.randn((2, 64, H, W), generator=gen)
    w = torch.randn((16, 64, 1, 1), generator=gen) * (2.0 / 64) ** 0.5
    y = F.conv2d(x, w, None, 2)
    dy = torch.randn(y.shape, generator=gen)
    g, dx, _, bx, _ = CG.reference(x, w, dy, 0, 1, y, stride=2)
    ex = CG.dgrad_stride2((dy * (y > 0).float()), w, H, W, prec, scatter)
    return G.check(ex, dx, bx, CG.apriori(prec, "dx", 64))


@pytest.mark.parametrize("hw", [(7, 9), (8, 6), (9, 10)])
@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_stride2_scatter(prec, hw):
    ok, r = _stride2(prec, *hw, "even")
    assert ok, r
    assert not _stride2(prec, *hw, "odd")[0]
    assert not _stride2(prec, *hw, "shift")[0]


# ------------------------------------------------------------------------------------------------
# forward (tests/test_gpu_conv_forward_fp64.py): conv_grad_oracle.forward's sums in fp32 pass the constant the GPU test
# uses, and each planted fault fails it
# ------------------------------------------------------------------------------------------------
def _fwd_layer(name):
    """(x, weight, kwargs) of a small layer: '3x3' 128 -> 192, N = 2 images of 7 x 9; 's2' 1x1 / stride 2, 64 -> 64 on
    9 x 11; 'up2' 1x1 64 -> 64 + a half-resolution residual on 8 x 10; 'res' 1x1 64 -> 64 + a residual + ReLU; 'head'
    the RPN's 1x1 A + 4A + A head (A = 3) with the sigmoid from channel 5A."""
    gen = torch.Generator().manual_seed(len(name))
    cin, cout, k, (H, W) = {"3x3": (128, 192, 3, (7, 9)), "s2": (64, 64, 1, (9, 11)), "up2": (64, 64, 1, (8, 10)),
                            "res": (64, 64, 1, (7, 9)), "head": (64, 18, 1, (7, 9))}[name]
    x = torch.randn((2, cin, H, W), generator=gen)
    w = torch.randn((cout, cin, k, k), generator=gen) * (2.0 / (cin * k * k)) ** 0.5
    kw = dict(bias=torch.randn(cout, generator=gen) * 0.5, padding=k // 2, relu=name in ("3x3", "res"))
    if name == "s2":
        kw["stride"] = 2
    if name == "up2":
        kw.update(residual=torch.randn((2, cout, H // 2, W // 2), generator=gen), residual_up2=True)
    if name == "res":
        kw["residual"] = torch.randn((2, cout, H, W), generator=gen)
    if name == "head":
        kw["sigmoid_from"] = 15
    return x, w, kw


def _fwd_check(prec, name, fault=None, pair=False):
    x, w, kw = _fwd_layer(name)
    if pair:
        x = CG.split(x)
    want, bound, slack = CG.forward(x, w, prec=prec, **kw)
    got, _, _ = CG.forward(x, w, prec=prec, fault=fault, dtype=torch.float32, **kw)
    K = w.shape[1] * w.shape[2] * w.shape[3]
    c = CG.forward_c(prec, K, int(kw.get("bias") is not None) + int(kw.get("residual") is not None))
    return G.check(got, want, bound, c, slack=slack)


FWD_LAYERS = ["3x3", "s2", "up2", "res", "head"]


@pytest.mark.parametrize("name", FWD_LAYERS)
@pytest.mark.parametrize("prec", ["bf16x3", "bf16", "fp32"])
def test_forward_restatement_passes(prec, name):
    ok, r = _fwd_check(prec, name)
    assert ok, r
    if prec == "bf16x3":
        ok, r = _fwd_check(prec, name, pair=True)
        assert ok, r


FWD_FAULTS = [("shift", "3x3"), ("stacked", "3x3"), ("drop_kblock", "3x3"), ("tile_from", "3x3"), ("odd", "s2"),
              ("up2_off", "up2"), ("bias_next", "res"), ("sigmoid_early", "head"), ("relu_first", "res")]


@pytest.mark.parametrize("fault", FWD_FAULTS, ids=[f for f, _ in FWD_FAULTS])
@pytest.mark.parametrize("prec", ["bf16x3", "bf16", "fp32"])
def test_forward_fault_fails(prec, fault):
    assert not _fwd_check(prec, fault[1], fault[0])[0]


@pytest.mark.parametrize("name", ["3x3", "s2"])
def test_forward_dropped_lohi_fails(name):
    assert not _fwd_check("bf16x3", name, "drop_lohi")[0]


@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_forward_truncated_split_fails(prec):
    assert not _fwd_check(prec, "s2", "trunc")[0]
