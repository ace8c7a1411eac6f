"""The window deformable conv (csrc/dcn_win.cu) with both output-channel tiles: N = 128 (two consumer warpgroups, K = 32
stages) and N = 32 (one consumer warpgroup, K = 64 stages), forced through upsnet_dcn_set_tile_n in one process.  Each
result is checked against the CPU oracle (oracle.deform_conv), and the two tiles against each other: every output element
sums the same K = 16 slices in the same order in both, so they must agree bit for bit.
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
    from upsnet_b200._lib import lib
    U.set_precision("bf16x3")
    was = dict(ops.DCN_WINDOW)
    ops.DCN_WINDOW.update(on=True, min_pixels=0)
    yield U
    assert lib().upsnet_dcn_set_tile_n(0) == 0
    ops.DCN_WINDOW.update(was)
    U.set_precision("fp32")


def t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _offsets(rng, kind, N, Ho, Wo):
    if kind == "small":
        return (rng.standard_normal((N, 18, Ho, Wo)) * 0.7).astype(np.float32)
    if kind == "tapbias":      # per-tap constant + small per-pixel part, broadcast over the batch
        o = rng.standard_normal((1, 18, 1, 1)) * 1.5 + rng.standard_normal((N, 18, Ho, Wo)) * 0.5
        return np.ascontiguousarray(o).astype(np.float32)
    if kind == "large":        # window centred on the mean sample, many corners gathered from global memory
        return (rng.standard_normal((N, 18, Ho, Wo)) * 6.0).astype(np.float32)
    if kind == "huge":         # most samples leave the window, many leave the image
        return (rng.standard_normal((N, 18, Ho, Wo)) * 25.0).astype(np.float32)
    raise ValueError(kind)


CASES = [
    # N, Cin, Cout, H, W, pad/dil, offsets, v2 mask
    dict(N=1, Cin=256, Cout=128, H=128, W=256, pd=1, off="tapbias", mask=False),   # semantic-head layer 0, 256 tiles
    dict(N=1, Cin=128, Cout=128, H=128, W=256, pd=1, off="tapbias", mask=True),    # semantic-head layer 1
    dict(N=1, Cin=256, Cout=256, H=40, W=72, pd=1, off="small", mask=False),       # two N tiles of 128
    dict(N=1, Cin=512, Cout=512, H=24, W=40, pd=1, off="tapbias", mask=True),      # four N tiles, 144 k-blocks of K = 32
    dict(N=3, Cin=128, Cout=128, H=45, W=70, pd=1, off="large", mask=False),       # batch 3, ragged tiles, outliers
    dict(N=1, Cin=128, Cout=128, H=40, W=64, pd=1, off="huge", mask=True),         # almost everything is an outlier
    dict(N=2, Cin=64, Cout=128, H=33, W=50, pd=2, off="small", mask=True),         # dilation 2, 9 k-blocks per sub-chunk pair
    dict(N=1, Cin=128, Cout=64, H=32, W=48, pd=1, off="tapbias", mask=False),      # Cout_pad 64: N = 32 only
    dict(N=1, Cin=128, Cout=192, H=32, W=48, pd=1, off="small", mask=False),       # Cout_pad 192: N = 32 only
    dict(N=1, Cin=64, Cout=16, H=20, W=20, pd=1, off="large", mask=True),          # Cout padded to 32: N = 32 only
]


def _run(U, ops, xp, off, w, b, mask, pd, dev):
    return U.deform_conv(xp, t(off, dev), t(w, dev), t(b, dev), 1, pd, pd, 1, mask=None if mask is None else t(mask, dev),
                         relu=False, precision=X3)


@pytest.mark.parametrize("cfg", CASES)
def test_wide_and_narrow_tiles_vs_oracle(dev, pair_mode, cfg):
    U = pair_mode
    from upsnet_b200 import operators as ops
    from upsnet_b200._lib import lib
    rng = np.random.default_rng(7)
    N, Cin, Cout, H, W, pd = cfg["N"], cfg["Cin"], cfg["Cout"], cfg["H"], cfg["W"], cfg["pd"]
    x = rng.standard_normal((N, Cin, H, W)).astype(np.float32)
    w = (rng.standard_normal((Cout, Cin, 3, 3)) / np.sqrt(Cin * 9)).astype(np.float32)
    b = rng.standard_normal(Cout).astype(np.float32)
    off = _offsets(rng, cfg["off"], N, H, W)
    mask = rng.uniform(0, 2, (N, 9, H, W)).astype(np.float32) if cfg["mask"] else None
    want = O.deform_conv(x, off, w, b, mask, 1, pd, pd, 1)
    xp = ops.Pair.from_float(t(x, dev))
    got = {}
    for bn in (128, 32):
        assert lib().upsnet_dcn_set_tile_n(bn) == 0
        l0 = ops.STATS["launches"]
        y = _run(U, ops, xp, off, w, b, mask, pd, dev)
        assert isinstance(y, ops.Pair) and ops.STATS["launches"] > l0
        got[bn] = y.float().cpu().numpy()
        err = np.abs(got[bn] - want).max()
        assert err < 1e-4, (bn, err)
    assert np.array_equal(got[128], got[32])


def test_tile_setter_rejects_other_values(dev):
    from upsnet_b200._lib import lib
    assert lib().upsnet_dcn_set_tile_n(64) == -1
    assert lib().upsnet_dcn_set_tile_n(0) == 0
