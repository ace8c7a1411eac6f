"""GPU parity of the window-staged deformable convolution on the pair stream (csrc/dcn_win.cu, upsnet_dcn_pair_forward)
against the CPU oracle (oracle.deform_conv: deform_conv_kernel.cu:89-118,194-242 restated) and against the global-gather
kernel it replaces (igemm_tc_kernel<1,2>).  The cases steer the per-tile sample statistics through every branch of the
kernel: all corners inside the bounding-box window (small offsets), window centred on the mean with outliers gathered
from global memory (large offsets), samples outside the image, ragged / small tiles (8x8 and 8x4 pixel blocks), all
N-tile shapes (Cout 16 .. 512), odd and even k-block counts (Cin 64 .. 512), v2 masks, ReLU.
Own file = own process (a trap in a tensor-core kernel poisons the CUDA context)."""
import numpy as np
import pytest
import torch

from oracle import oracle as O

pytestmark = pytest.mark.gpu
X3 = 1


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


@pytest.fixture()
def pair_mode():
    import upsnet_b200 as U
    from upsnet_b200 import operators as ops
    U.set_precision("bf16x3")
    was = dict(ops.DCN_WINDOW)
    ops.DCN_WINDOW.update(on=True, min_pixels=0)
    yield U
    ops.DCN_WINDOW.update(was)
    U.set_precision("fp32")


def t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _case(rng, N, Cin, Cout, H, W):
    x = rng.standard_normal((N, Cin, H, W)).astype(np.float32)
    w = (rng.standard_normal((Cout, Cin, 3, 3)) / np.sqrt(Cin * 9)).astype(np.float32)
    b = rng.standard_normal(Cout).astype(np.float32)
    return x, w, b


def _offsets(rng, kind, N, Ho, Wo):
    if kind == "small":        # everything inside the bounding-box window
        return (rng.standard_normal((N, 18, Ho, Wo)) * 0.7).astype(np.float32)
    if kind == "tapbias":      # the synthetic model's structure: per-tap constant + small per-pixel part
        return (rng.standard_normal((1, 18, 1, 1)) * 1.5 + rng.standard_normal((N, 18, Ho, Wo)) * 0.5).astype(np.float32)
    if kind == "large":        # window centred on the mean, many outliers
        return (rng.standard_normal((N, 18, Ho, Wo)) * 6.0).astype(np.float32)
    if kind == "huge":         # most samples leave the window, many leave the image
        return (rng.standard_normal((N, 18, Ho, Wo)) * 25.0).astype(np.float32)
    if kind == "zero":
        return np.zeros((N, 18, Ho, Wo), np.float32)
    raise ValueError(kind)


CASES = [
    # N, Cin, Cout, H, W, pad/dil, offsets
    dict(N=1, Cin=256, Cout=128, H=32, W=48, pd=1, off="tapbias"),     # semantic-head layer 0 shape class (a12)
    dict(N=1, Cin=128, Cout=128, H=32, W=48, pd=1, off="small"),       # semantic-head layer 1
    dict(N=1, Cin=64, Cout=64, H=16, W=16, pd=1, off="small"),         # 9 k-blocks (odd): group parity alternates per tile
    dict(N=2, Cin=128, Cout=128, H=25, W=42, pd=1, off="large"),       # ragged tiles, batch, outliers
    dict(N=1, Cin=64, Cout=16, H=20, W=20, pd=2, off="small"),         # dilation 2, Cout padded to 64
    dict(N=1, Cin=256, Cout=256, H=24, W=40, pd=1, off="tapbias"),     # two N tiles (res4 DCN of config B)
    dict(N=1, Cin=512, Cout=512, H=13, W=21, pd=1, off="small"),       # four N tiles, 72 k-blocks (res5 DCN of config B)
    dict(N=1, Cin=128, Cout=128, H=8, W=16, pd=1, off="large"),        # single tile
    dict(N=1, Cin=128, Cout=128, H=40, W=64, pd=1, off="huge"),        # almost everything is an outlier / outside the image
    dict(N=1, Cin=64, Cout=64, H=6, W=5, pd=1, off="zero"),            # map smaller than a tile, zero offsets == dense conv
    dict(N=3, Cin=64, Cout=128, H=64, W=96, pd=1, off="tapbias"),      # > 132 tiles: persistent CTAs run several tiles
]


@pytest.mark.parametrize("modulated", [False, True])
@pytest.mark.parametrize("cfg", CASES)
def test_window_dcn_vs_oracle(dev, pair_mode, cfg, modulated):
    U = pair_mode
    from upsnet_b200 import operators as ops
    rng = np.random.default_rng(21)
    N, Cin, Cout, H, W, pd = cfg["N"], cfg["Cin"], cfg["Cout"], cfg["H"], cfg["W"], cfg["pd"]
    x, w, b = _case(rng, N, Cin, Cout, H, W)
    off = _offsets(rng, cfg["off"], N, H, W)
    off = np.ascontiguousarray(np.broadcast_to(off, (N, 18, H, W))) if off.shape != (N, 18, H, W) else off
    mask = rng.uniform(0, 2, (N, 9, H, W)).astype(np.float32) if modulated else None
    want = O.deform_conv(x, off, w, b, mask, 1, pd, pd, 1)
    xp = ops.Pair.from_float(t(x, dev))
    assert ops.DCN_WINDOW["on"]
    launches0 = ops.STATS["launches"]
    got = U.deform_conv(xp, t(off, dev), t(w, dev), t(b, dev), 1, pd, pd, 1, mask=None if mask is None else t(mask, dev),
                        relu=False, precision=X3)
    assert isinstance(got, ops.Pair) and ops.STATS["launches"] > launches0
    g = got.float().cpu().numpy()
    err = np.abs(g - want).max()
    assert err < 1e-4, err
    # and against the global-gather kernel this one replaces (same contract, different K order -> fp32 rounding only)
    ops.DCN_WINDOW["on"] = False
    try:
        ref = U.deform_conv(xp, t(off, dev), t(w, dev), t(b, dev), 1, pd, pd, 1, mask=None if mask is None else t(mask, dev),
                            relu=False, precision=X3)
    finally:
        ops.DCN_WINDOW["on"] = True
    assert np.abs(ref.float().cpu().numpy() - g).max() < 1e-4


def test_window_dcn_relu_and_module(dev, pair_mode):
    """DeformConvWithOffset on a Pair (models/fcn.py:40-55 shape class): offset conv + window DCN + ReLU."""
    U = pair_mode
    from upsnet_b200 import operators as ops
    rng = np.random.default_rng(5)
    x, w, b = _case(rng, 1, 128, 128, 24, 36)
    off = _offsets(rng, "tapbias", 1, 24, 36)
    off = np.ascontiguousarray(np.broadcast_to(off, (1, 18, 24, 36)))
    want = np.maximum(O.deform_conv(x, off, w, b, None, 1, 1, 1, 1), 0)
    got = U.deform_conv(ops.Pair.from_float(t(x, dev)), t(off, dev), t(w, dev), t(b, dev), 1, 1, 1, 1, relu=True, precision=X3)
    assert np.abs(got.float().cpu().numpy() - want).max() < 1e-4


def test_window_dcn_c_abi_rejects_other_shapes(dev):
    import ctypes as C
    from upsnet_b200._lib import lib
    nb = C.c_size_t(0)
    assert lib().upsnet_dcn_packed_weight_bytes(128, 256, 3, 3, C.byref(nb)) == 0 and nb.value == 2 * 128 * 9 * 256 * 2
    assert lib().upsnet_dcn_packed_weight_bytes(128, 256, 1, 1, C.byref(nb)) == -2      # 3x3 only
    assert lib().upsnet_dcn_packed_weight_bytes(128, 96, 3, 3, C.byref(nb)) == -2       # Cin % 64
    assert lib().upsnet_dcn_packed_weight_bytes(20, 64, 3, 3, C.byref(nb)) == 0 and nb.value == 2 * 32 * 9 * 64 * 2   # rows padded to 32
