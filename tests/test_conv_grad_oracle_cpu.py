"""CPU check that the bounds of tests/test_gpu_conv_backward.py have teeth: a torch restatement of the dense-conv
backward arithmetic (tests/conv_grad_oracle.py: hi/lo pairs or bf16 operands, flipped-tap dgrad, per-tap wgrad over K
splits) passes grad_oracle.check at the a-priori constants, and each planted fault fails it: a tap not flipped, x read
one pixel off, one K split dropped, the ReLU mask missing."""
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
