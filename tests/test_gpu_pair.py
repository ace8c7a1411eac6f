"""GPU parity of the hi/lo bf16 PAIR activation stream (precision bf16x3 on the TMA-fed wgmma kernel):
every layer shape class of the engine against the CPU oracle at the "fp32 logits within 1e-3" contract -- in practice
held to ~1e-5 relative, which is what makes the pair stream an fp32-grade format.  Own file = own process (a trap in a
tensor-core kernel poisons the CUDA context)."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from kernel_trace import launched_kernels  # noqa: E402

pytestmark = pytest.mark.gpu
X3 = 1


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


@pytest.fixture()
def pair_mode():
    import upsnet_b200 as U
    U.set_precision("bf16x3")
    yield U
    U.set_precision("fp32")


def t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _case(rng, N, Cin, Cout, H, W, k):
    x = rng.standard_normal((N, Cin, H, W)).astype(np.float32)
    w = (rng.standard_normal((Cout, Cin, k, k)) / np.sqrt(Cin * k * k)).astype(np.float32)
    b = rng.standard_normal(Cout).astype(np.float32)
    return x, w, b


def _bound(x, w, stride, pad, dil):
    """Element-wise error scale of a dot product: sum |x||w| (the 3-term split loses ~2^-16 of it at worst)."""
    return O.conv2d(np.abs(x), np.abs(w), None, stride, pad, dil)


def test_pair_roundtrip(dev, pair_mode):
    from upsnet_b200.operators import Pair
    x = torch.randn(2, 64, 9, 11, device=dev) * 37.0
    p = Pair.from_float(x)
    assert p.shape == x.shape and p.store.shape == (2, 9, 11, 128)
    err = (p.float() - x).abs().max().item()
    assert err <= 2.0 ** -16 * x.abs().max().item(), err


def _conv_kernels(fn):
    """fn() under torch.profiler: its result and the names of the implicit-GEMM conv kernels it launched
    (tests/kernel_trace.py: sessions that lost their records are repeated)."""
    return launched_kernels(fn, lambda n: "igemm_" in n)


def _assert_kernel(names, tma):
    """The TMA-fed kernel serves the layer when it is enabled (no silent fall-back to the gather kernel), else the gather one."""
    want, other = ("igemm_tma_kernel", "igemm_tc_kernel") if tma else ("igemm_tc_kernel", "igemm_tma_kernel")
    assert any(want in n for n in names) and not any(other in n for n in names), names


CONV_CASES = [
    dict(N=1, Cin=64, Cout=64, H=16, W=16, k=1, stride=1, pad=0, dil=1),      # one k-block
    dict(N=1, Cin=256, Cout=64, H=16, W=24, k=1, stride=1, pad=0, dil=1),     # ring wrap
    dict(N=1, Cin=64, Cout=128, H=20, W=28, k=3, stride=1, pad=1, dil=1),     # 3x3, ragged tiles
    dict(N=1, Cin=256, Cout=256, H=32, W=48, k=3, stride=1, pad=1, dil=1),    # FPN / RPN 3x3 shape class
    dict(N=2, Cin=128, Cout=256, H=15, W=17, k=3, stride=1, pad=1, dil=1),    # batch, odd sizes
    dict(N=1, Cin=256, Cout=512, H=16, W=20, k=1, stride=2, pad=0, dil=1),    # strided 1x1 (down-sampling conv)
    dict(N=1, Cin=64, Cout=256, H=24, W=40, k=1, stride=1, pad=0, dil=1),     # res2 conv3 (+res: in-place slab pairs)
    dict(N=1, Cin=512, Cout=512, H=8, W=16, k=3, stride=1, pad=1, dil=1),     # res5 conv2: many k-blocks, few tiles
    dict(N=1, Cin=128, Cout=128, H=14, W=14, k=3, stride=1, pad=2, dil=2),    # dilation
    dict(N=12, Cin=256, Cout=256, H=14, W=14, k=3, stride=1, pad=1, dil=1),   # mask-head roi batch (boxes span images)
    dict(N=50, Cin=1024, Cout=1024, H=1, W=1, k=1, stride=1, pad=0, dil=1),   # fc7
    dict(N=37, Cin=12544, Cout=1024, H=1, W=1, k=1, stride=1, pad=0, dil=1),  # fc6 (196 k-blocks)
]


@pytest.mark.parametrize("cfg", CONV_CASES)
@pytest.mark.parametrize("tma", [True, False])
def test_pair_conv_vs_oracle(dev, pair_mode, cfg, tma):
    """Pair in -> pair out, with and without bias / residual / ReLU; TMA kernel and the cp.async gather kernel."""
    U = pair_mode
    from upsnet_b200 import operators as ops
    from upsnet_b200.operators import Pair
    rng = np.random.default_rng(11)
    x, w, b = _case(rng, cfg["N"], cfg["Cin"], cfg["Cout"], cfg["H"], cfg["W"], cfg["k"])
    want = O.conv2d(x, w, b, cfg["stride"], cfg["pad"], cfg["dil"])
    bound = _bound(x, w, cfg["stride"], cfg["pad"], cfg["dil"])
    res = rng.standard_normal(want.shape).astype(np.float32)
    ops.USE_TMA["on"] = tma
    try:
        xp = Pair.from_float(t(x, dev))
        got, k1 = _conv_kernels(lambda: U.conv2d(xp, t(w, dev), t(b, dev), cfg["stride"], cfg["pad"], cfg["dil"], precision=X3))
        _assert_kernel(k1, tma)
        assert isinstance(got, Pair) and got.shape == want.shape
        g = got.float().cpu().numpy()
        # 3 MMAs drop only lo*lo (2^-18 of sum|x||w|); pair storage of x and y adds 2^-17 each
        err = np.abs(g - want)
        assert (err <= 4e-5 * bound + 2e-5 * np.abs(want) + 1e-6).all(), float((err / (bound + 1e-3)).max())
        assert err.max() < 1e-3
        rp = Pair.from_float(t(res, dev))
        got2, k2 = _conv_kernels(lambda: U.conv2d(xp, t(w, dev), t(b, dev), cfg["stride"], cfg["pad"], cfg["dil"], residual=rp,
                                                  relu=True, precision=X3))
        _assert_kernel(k2, tma)
        want2 = np.maximum(want + res, 0)
        err2 = np.abs(got2.float().cpu().numpy() - want2)
        assert (err2 <= 4e-5 * bound + 4e-5 * (np.abs(want) + np.abs(res)) + 1e-6).all(), float(err2.max())
        # fp32 plane-wise head output from a pair input (direct-store epilogue), Cout clipped to a head-like count
        co = min(cfg["Cout"], 19)
        got3, k3 = _conv_kernels(lambda: U.conv2d(xp, t(w[:co].copy(), dev), t(b[:co].copy(), dev), cfg["stride"], cfg["pad"],
                                                  cfg["dil"], precision=X3, out_format="nchw"))
        _assert_kernel(k3, tma)
        assert got3.dtype == torch.float32 and got3.is_contiguous()
        err3 = np.abs(got3.cpu().numpy() - want[:, :co])
        assert (err3 <= 4e-5 * bound[:, :co] + 1e-6).all(), float(err3.max())
    finally:
        ops.USE_TMA["on"] = True


def test_pair_fpn_lateral_up2(dev, pair_mode):
    """Lateral 1x1 + nearest-2x-upsampled coarser pair map fused in the epilogue (models/fpn.py:88-93)."""
    U = pair_mode
    from upsnet_b200.operators import Pair
    rng = np.random.default_rng(12)
    for (H, W, Cin) in ((16, 24, 256), (32, 64, 512)):
        x, w, b = _case(rng, 1, Cin, 256, H, W, 1)
        coarse = rng.standard_normal((1, 256, H // 2, W // 2)).astype(np.float32)
        want = O.conv2d(x, w, b) + coarse.repeat(2, axis=2).repeat(2, axis=3)
        got = U.conv2d(Pair.from_float(t(x, dev)), t(w, dev), t(b, dev), residual=Pair.from_float(t(coarse, dev)),
                       residual_up2=True, precision=X3)
        err = np.abs(got.float().cpu().numpy() - want).max()
        assert err < 2e-4, err


def test_pair_group_deconv_commute(dev, pair_mode):
    """1x1 conv to 4*Cout channels written as four [hi Cout][lo Cout] groups == the Pair of 4w pixels per row."""
    U = pair_mode
    from upsnet_b200.operators import Pair
    rng = np.random.default_rng(13)
    x, w, b = _case(rng, 6, 256, 1024, 14, 14, 1)
    want = np.maximum(O.conv2d(x, w, b), 0)                                  # [n, 1024, h, w]
    got = U.conv2d(Pair.from_float(t(x, dev)), t(w, dev), t(b, dev), relu=True, precision=X3, pair_group=256)
    assert got.shape == (6, 256, 14, 56)
    g = got.float().cpu().numpy()                                            # [n, 256, h, 4w]: pixel index = w*4 + group
    w_ = want.reshape(6, 4, 256, 14, 14).transpose(0, 2, 3, 4, 1).reshape(6, 256, 14, 56)
    assert np.abs(g - w_).max() < 2e-4


@pytest.mark.parametrize("modulated", [False, True])
@pytest.mark.parametrize("cfg", [
    dict(N=1, Cin=64, Cout=64, H=16, W=16, stride=1, pad=1, dil=1),
    dict(N=1, Cin=256, Cout=128, H=32, W=48, stride=1, pad=1, dil=1),         # semantic-head layer shape (a12)
    dict(N=2, Cin=128, Cout=128, H=25, W=42, stride=1, pad=1, dil=1),         # ragged (config B 25x42)
    dict(N=1, Cin=64, Cout=64, H=20, W=20, stride=1, pad=2, dil=2),
])
def test_pair_dcn_vs_oracle(dev, pair_mode, cfg, modulated):
    U = pair_mode
    from upsnet_b200.operators import Pair
    rng = np.random.default_rng(6)
    N, Cin, Cout, H, W = cfg["N"], cfg["Cin"], cfg["Cout"], cfg["H"], cfg["W"]
    Ho = O.conv_out(H, cfg["pad"], cfg["dil"], 3, cfg["stride"]); Wo = O.conv_out(W, cfg["pad"], cfg["dil"], 3, cfg["stride"])
    x, w, b = _case(rng, N, Cin, Cout, H, W, 3)
    off = (rng.standard_normal((N, 18, Ho, Wo)) * 2.5).astype(np.float32)
    mask = rng.uniform(0, 2, (N, 9, Ho, Wo)).astype(np.float32) if modulated else None
    want = O.deform_conv(x, off, w, b, mask, cfg["stride"], cfg["pad"], cfg["dil"], 1)
    got = U.deform_conv(Pair.from_float(t(x, dev)), t(off, dev), t(w, dev), t(b, dev), cfg["stride"], cfg["pad"], cfg["dil"], 1,
                        mask=None if mask is None else t(mask, dev), relu=False, precision=X3)
    assert isinstance(got, Pair)
    err = np.abs(got.float().cpu().numpy() - want).max()
    assert err < 1e-4, err


def test_pair_stem_maxpool(dev, pair_mode):
    """RGB stem (7x7/2 on the fp32 image) -> Pair, then the 3x3/2 max-pool on pairs (models/resnet.py:155-163)."""
    U = pair_mode
    from upsnet_b200 import operators as ops
    rng = np.random.default_rng(14)
    x = (rng.standard_normal((1, 3, 64, 96)) * 60).astype(np.float32)
    w = (rng.standard_normal((64, 3, 7, 7)) / 12).astype(np.float32)
    b = rng.standard_normal(64).astype(np.float32)
    y = U.conv2d(t(x, dev), t(w, dev), t(b, dev), 2, 3, 1, relu=True, precision=X3)
    assert isinstance(y, ops.Pair)
    want = np.maximum(O.conv2d(x, w, b, 2, 3, 1), 0)
    yf = y.float()
    assert np.abs(yf.cpu().numpy() - want).max() < 1e-3 * max(1.0, np.abs(want).max())
    mp = ops.max_pool2d(y, 3, 2, 1)
    ref = torch.nn.functional.max_pool2d(yf, 3, 2, 1)
    assert torch.equal(mp.float(), ref)               # the winning (hi, lo) is copied verbatim


def test_pair_stem_tma(dev, pair_mode):
    """The TMA-fed stem on hi/lo copies of the image (upsnet_stem_forward + UPSNET_EPI_STEM_PAIR) == the gather stem == oracle."""
    U = pair_mode
    from upsnet_b200 import operators as ops
    rng = np.random.default_rng(16)
    for (H, W) in ((64, 96), (224, 320)):
        x = (rng.standard_normal((1, 3, H, W)) * 60).astype(np.float32)
        w = (rng.standard_normal((64, 3, 7, 7)) / 12).astype(np.float32)
        b = rng.standard_normal(64).astype(np.float32)
        y = ops.stem_conv(t(x, dev), t(w, dev), t(b, dev), 3, relu=True, pair=True)
        assert isinstance(y, ops.Pair) and y.shape == (1, 64, H // 2, W // 2)
        want = np.maximum(O.conv2d(x, w, b, 2, 3, 1), 0)
        err = np.abs(y.float().cpu().numpy() - want).max()
        assert err < 2e-4 * max(1.0, np.abs(want).max()), err


def test_pair_fpn_roi_align(dev, pair_mode):
    """Pair ROIAlign (pair pixels and the flat fc6 layout) == the fp32 kernel on hi + lo, to pair rounding."""
    U = pair_mode
    from upsnet_b200 import operators as ops
    rng = np.random.default_rng(15)
    feats = [torch.randn(1, 256, 64 >> l, 96 >> l, device=dev) for l in range(4)]
    pairs = [ops.Pair.from_float(f) for f in feats]
    exact = [p.float().contiguous() for p in pairs]
    n = 40
    c = rng.uniform(0, 1, (n, 2)) * np.array([380, 250]); s = np.exp(rng.uniform(np.log(8), np.log(300), (n, 2)))
    rois = np.concatenate([np.zeros((n, 1)), np.clip(c - s / 2, 0, [383, 255]), np.clip(c + s / 2, 0, [383, 255])], 1).astype(np.float32)
    sc = [1 / 4., 1 / 8., 1 / 16., 1 / 32.]
    for ph in (7, 14):
        want = U.fpn_roi_align(exact, t(rois, dev), ph, ph, sc)                      # fp32 NCHW kernel
        got = U.fpn_roi_align(pairs, t(rois, dev), ph, ph, sc, layout="auto")
        assert isinstance(got, ops.Pair) and got.shape == want.shape
        assert (got.float() - want).abs().max().item() < 2e-5 * max(1.0, want.abs().max().item())
    flat = U.fpn_roi_align(pairs, t(rois, dev), 7, 7, sc, layout="flat_pair")
    assert flat.shape == (n, 49 * 256, 1, 1)
    want = U.fpn_roi_align(exact, t(rois, dev), 7, 7, sc).permute(0, 2, 3, 1).reshape(n, -1)
    assert (flat.float().reshape(n, -1) - want).abs().max().item() < 2e-5 * max(1.0, want.abs().max().item())


def test_engine_pair_stream_vs_fp32(dev):
    """The whole engine in the pair stream (bf16x3) vs the fp32 CUDA-core path: semantic logits within 1e-3, label maps
    equal wherever the top-2 logit margin is not tiny."""
    import upsnet_b200 as U
    from upsnet_b200.model import UPSNetConfig
    from upsnet_b200.synthetic import synthetic_input, synthetic_model
    m = synthetic_model(UPSNetConfig.cityscapes_r50(), depth=(2, 2, 2, 2), seed=5, device=dev)
    m.keep_intermediates = True
    inp = synthetic_input(256, 384, seed=6, device=dev)
    outs = {}
    try:
        for name in ("fp32", "bf16x3"):
            U.set_precision(name)
            with torch.no_grad():
                outs[name] = m(inp)
    finally:
        U.set_precision("fp32")
    ref = outs["fp32"]["_intermediates"]["fcn_output"].float()
    scale = max(1.0, float(ref.abs().max()))
    d = (outs["bf16x3"]["_intermediates"]["fcn_output"].float() - ref).abs().max().item()
    assert d <= 1e-3 * scale, (d, scale)
    agree = (outs["bf16x3"]["fcn_outputs"] == outs["fp32"]["fcn_outputs"]).float().mean().item()
    assert agree > 0.999, agree
    assert outs["bf16x3"]["panoptic_outputs"].shape == outs["fp32"]["panoptic_outputs"].shape
