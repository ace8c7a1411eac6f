"""The TMA-fed dense conv (csrc/igemm_tma.cu) on hi/lo pairs with both output-channel tiles: N = 128 (one m64n256 wgmma over
[W_hi ; W_lo] plus one m64n128 per K slice) and N = 64 (m64n128 + m64n64), forced through upsnet_tma_set_tile_n in one
process.  Each result is checked against a reference at the pair-stream tolerance of test_gpu_pair.py, and the two tiles
against each other: every output element goes through the same MMAs and additions in the same order in both, so the
stored (hi, lo) pairs must agree bit for bit.  Layers whose N = 128 tile does not fit (in-place residual slabs, FPN
up-sampled residual) must fall back to N = 64 and still match.
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
    from upsnet_b200._lib import lib
    U.set_precision("bf16x3")
    yield U
    assert lib().upsnet_tma_set_tile_n(0) == 0
    U.set_precision("fp32")


def t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _case(rng, N, Cin, Cout, H, W, k):
    x = rng.standard_normal((N, Cin, H, W)).astype(np.float32)
    w = (rng.standard_normal((Cout, Cin, k, k)) / np.sqrt(Cin * k * k)).astype(np.float32)
    b = rng.standard_normal(Cout).astype(np.float32)
    return x, w, b


def _tma_kernels(fn):
    """fn() under torch.profiler: its result and the names of the conv kernels it launched."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, {e.key for e in prof.key_averages() if "igemm_" in e.key}


def _wide(names):
    """True when the N = 128 pair tile ran (instance <256, 1>), False for N = 64 (<128, 1>).  None when the profiler
    session reported no kernel records at all, which it occasionally does: the results are still checked then."""
    if not names:
        return None
    tma = [n for n in names if "igemm_tma_kernel" in n]
    w = [n for n in tma if "<256, 1>" in n or "<256,1>" in n]
    n = [n for n in tma if "<128, 1>" in n or "<128,1>" in n]
    assert bool(w) != bool(n), sorted(names)
    return bool(w)


def _both_tiles(fn):
    """fn() with the N tile forced to 128, then to 64: {bn: (result, ran the N = 128 instance)}."""
    from upsnet_b200._lib import lib
    out = {}
    for bn in (128, 64):
        assert lib().upsnet_tma_set_tile_n(bn) == 0
        y, names = _tma_kernels(fn)
        out[bn] = (y, _wide(names))
    assert lib().upsnet_tma_set_tile_n(0) == 0
    return out


def _check(got, want, bound):
    err = np.abs(got - want)
    assert (err <= 4e-5 * bound + 2e-5 * np.abs(want) + 1e-6).all(), float((err / (bound + 1e-3)).max())
    assert err.max() < 1e-3


# test_gpu_pair.CONV_CASES with Cout % 128 == 0
CASES = [
    dict(N=1, Cin=64, Cout=128, H=20, W=28, k=3, stride=1, pad=1, dil=1),     # 3x3, ragged tiles
    dict(N=1, Cin=256, Cout=256, H=32, W=48, k=3, stride=1, pad=1, dil=1),    # FPN / RPN 3x3 shape class
    dict(N=2, Cin=128, Cout=256, H=15, W=17, k=3, stride=1, pad=1, dil=1),    # batch, odd sizes
    dict(N=1, Cin=256, Cout=512, H=16, W=20, k=1, stride=2, pad=0, dil=1),    # strided 1x1 (down-sampling conv)
    dict(N=1, Cin=64, Cout=256, H=24, W=40, k=1, stride=1, pad=0, dil=1),     # res2 conv3
    dict(N=1, Cin=512, Cout=512, H=8, W=16, k=3, stride=1, pad=1, dil=1),     # res5 conv2: many k-blocks, few tiles
    dict(N=1, Cin=128, Cout=128, H=14, W=14, k=3, stride=1, pad=2, dil=2),    # dilation
    dict(N=12, Cin=256, Cout=256, H=14, W=14, k=3, stride=1, pad=1, dil=1),   # mask-head roi batch (boxes span images)
    dict(N=50, Cin=1024, Cout=1024, H=1, W=1, k=1, stride=1, pad=0, dil=1),   # fc7
    dict(N=37, Cin=12544, Cout=1024, H=1, W=1, k=1, stride=1, pad=0, dil=1),  # fc6 (196 k-blocks)
]


@pytest.mark.parametrize("cfg", CASES)
def test_wide_and_narrow_tiles_vs_oracle(dev, pair_mode, cfg):
    """No residual: N = 128 runs when forced; with bias + ReLU; the residual form falls back to N = 64 and matches."""
    U = pair_mode
    from upsnet_b200.operators import Pair
    rng = np.random.default_rng(11)
    x, w, b = _case(rng, cfg["N"], cfg["Cin"], cfg["Cout"], cfg["H"], cfg["W"], cfg["k"])
    s, p, d = cfg["stride"], cfg["pad"], cfg["dil"]
    want = O.conv2d(x, w, b, s, p, d)
    bound = O.conv2d(np.abs(x), np.abs(w), None, s, p, d)
    xp = Pair.from_float(t(x, dev))
    runs = _both_tiles(lambda: U.conv2d(xp, t(w, dev), t(b, dev), s, p, d, relu=True, precision=X3))
    assert runs[128][1] in (True, None) and runs[64][1] in (False, None)
    for bn in (128, 64):
        _check(runs[bn][0].float().cpu().numpy(), np.maximum(want, 0), bound)
    assert torch.equal(runs[128][0].store, runs[64][0].store)
    # in-place residual slab pairs need 128 KB at N = 128: the forced tile falls back to 64
    res = rng.standard_normal(want.shape).astype(np.float32)
    rp = Pair.from_float(t(res, dev))
    runs = _both_tiles(lambda: U.conv2d(xp, t(w, dev), t(b, dev), s, p, d, residual=rp, relu=True, precision=X3))
    assert runs[128][1] in (False, None) and runs[64][1] in (False, None)
    want2 = np.maximum(want + res, 0)
    err2 = np.abs(runs[128][0].float().cpu().numpy() - want2)
    assert (err2 <= 4e-5 * bound + 4e-5 * (np.abs(want) + np.abs(res)) + 1e-6).all(), float(err2.max())
    assert torch.equal(runs[128][0].store, runs[64][0].store)


def _ref64(x, w, b, pad):
    """fp64 reference on the device for the full-size shapes (the CPU oracle would take minutes at these sizes)."""
    return torch.nn.functional.conv2d(x.double(), w.double(), b.double(), padding=pad)


@pytest.mark.parametrize("shape", [(1, 256, 256, 512), (256, 256, 14, 14)], ids=["fpn_3x3_256x512", "mask_head_256_rois"])
def test_full_size_3x3(dev, pair_mode, shape):
    """The FPN / RPN 3x3 at 256x512 and the mask-head batch of 256 rois of 14x14, both tiles vs fp64, bit-identical."""
    U = pair_mode
    from upsnet_b200.operators import Pair
    N, C, H, W = shape
    g = torch.Generator(device=dev).manual_seed(3)
    x = torch.randn(N, C, H, W, device=dev, generator=g)
    w = torch.randn(256, C, 3, 3, device=dev, generator=g) / (C * 9) ** 0.5
    b = torch.randn(256, device=dev, generator=g)
    xp = Pair.from_float(x)
    want = _ref64(x, w, b, 1)
    bound = torch.nn.functional.conv2d(x.double().abs(), w.double().abs(), None, padding=1)
    runs = _both_tiles(lambda: U.conv2d(xp, w, b, 1, 1, 1, precision=X3))
    assert runs[128][1] in (True, None) and runs[64][1] in (False, None)
    for bn in (128, 64):
        err = (runs[bn][0].float().double() - want).abs()
        assert bool((err <= 4e-5 * bound + 2e-5 * want.abs() + 1e-6).all()), float(err.max())
    assert torch.equal(runs[128][0].store, runs[64][0].store)


def test_pair_group_deconv(dev, pair_mode):
    """1x1 conv to 4 x 256 channels stored as four [hi 256][lo 256] groups (the mask-head deconv), both tiles."""
    U = pair_mode
    from upsnet_b200.operators import Pair
    rng = np.random.default_rng(13)
    x, w, b = _case(rng, 6, 256, 1024, 14, 14, 1)
    want = np.maximum(O.conv2d(x, w, b), 0)
    w_ = want.reshape(6, 4, 256, 14, 14).transpose(0, 2, 3, 4, 1).reshape(6, 256, 14, 56)
    xp = Pair.from_float(t(x, dev))
    runs = _both_tiles(lambda: U.conv2d(xp, t(w, dev), t(b, dev), relu=True, precision=X3, pair_group=256))
    assert runs[128][1] in (True, None) and runs[64][1] in (False, None)
    for bn in (128, 64):
        assert runs[bn][0].shape == (6, 256, 14, 56)
        assert np.abs(runs[bn][0].float().cpu().numpy() - w_).max() < 2e-4
    assert torch.equal(runs[128][0].store, runs[64][0].store)


def test_fpn_lateral_up2_falls_back(dev, pair_mode):
    """Lateral 1x1 + nearest-2x up-sampled coarser map: N = 128 would leave a 2-stage ring, so a forced 128 runs at 64."""
    U = pair_mode
    from upsnet_b200.operators import Pair
    rng = np.random.default_rng(12)
    for (H, W, Cin) in ((16, 24, 256), (32, 64, 512)):
        x, w, b = _case(rng, 1, Cin, 256, H, W, 1)
        coarse = rng.standard_normal((1, 256, H // 2, W // 2)).astype(np.float32)
        want = O.conv2d(x, w, b) + coarse.repeat(2, axis=2).repeat(2, axis=3)
        xp, cp = Pair.from_float(t(x, dev)), Pair.from_float(t(coarse, dev))
        runs = _both_tiles(lambda: U.conv2d(xp, t(w, dev), t(b, dev), residual=cp, residual_up2=True, precision=X3))
        assert runs[128][1] in (False, None) and runs[64][1] in (False, None)
        assert np.abs(runs[128][0].float().cpu().numpy() - want).max() < 2e-4
        assert torch.equal(runs[128][0].store, runs[64][0].store)


def test_tile_setter_rejects_other_values(dev):
    from upsnet_b200._lib import lib
    assert lib().upsnet_tma_set_tile_n(32) == -1
    assert lib().upsnet_tma_set_tile_n(96) == -1
    assert lib().upsnet_tma_set_tile_n(0) == 0
