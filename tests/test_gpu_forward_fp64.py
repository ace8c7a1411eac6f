"""Forward kernels of the inference engine -- deformable convolution on the tensor-core paths (csrc/dcn_win.cu,
csrc/igemm_tc.cu) and ROIAlign in the NHWC fp32 / bf16 / pair layouts (csrc/roi_align.cu) -- against the float64
restatement of tests/grad_oracle.py run on the device, element by element, each element against its own bound:
|kernel - fp64| <= c * (sum of |terms|) + slack + 1e-6.  Sample positions come from grad_oracle.special_offsets (exact
fp32 positions on the integers, -1, H, ... where floor and the corner guards decide; `window` mode aims at the window
kernel's geometry), rois from grad_oracle.hand_rois.  Every DCN case asserts through the profiler which kernel ran.
Run with -s to see the worst err / bound per path.  Own file = own process (a trap in a tensor-core kernel poisons the
CUDA context).

Bounds (u = 2^-16; T = |bias| + sum over the Cin*9 terms of |weight| * bilinear(|x|) * mask, the bound tensor):

bf16x3 (three MMAs hi*hi + lo*hi + hi*lo; the reference gets the exact activation value hi + lo of a pair, or the fp32
activation).  Per term, relative to |weight| * bilinear(|x|) * mask:
  * the blend of the lo plane (pair activations only): bf16 corner weights and a bf16 FMA chain (HMUL2 + 3 HFMA2), one
    weight rounding and four chain roundings, each <= 2^-8 of a sum of |w lo| <= 2^-8 sum w |x|: 5 u.  The hi plane /
    fp32 activations are blended by four fp32 FMAs: 4 * 2^-24 = 0.06 u.
  * the blended sample split into bf16 hi / lo: |s - hi - lo| <= 2^-17 |s|: 0.5 u.  The weight split: 0.5 u.
  * lo * lo dropped: |s_lo w_lo| <= 2^-8 |s| 2^-8 |w|: 1 u.
  * fp32 accumulation: 3 K / 16 wgmma steps of exact products, each adding at most 2 * 2^-24 of the magnitudes (the
    tensor core aligns the addends by truncation): 3 K / 8 * 2^-24 = 6.75 u at the largest K here (9 * 512).
  Sum: 13.8 u = 2.1e-4 with pair activations, 8.8 u = 1.35e-4 with fp32 activations (grad_oracle.TOL "dcn_x3_pair",
  "dcn_x3_f32" before measurement).  A pair output adds hi = bf16(o), lo = bf16(o - hi): 2^-17 |o| (slack).
bf16 (bf16 activations, bf16-exact weights, one MMA).  The gather rounds inside its blend: the fp32 corner weight times
  the mask (the mask is applied before rounding) is rounded to bf16, then HMUL2 + 3 HFMA2, each rounded to bf16.  The
  reference (grad_oracle.dcn_columns mode 'bf16') repeats exactly these roundings in float64 (ties to even), so its
  samples equal the kernel's bit for bit and no slack for samples near a bf16 rounding midpoint is needed.  What is
  left is the fp32 accumulation, K / 16 steps: K / 8 * 2^-24 of T' = |bias| + sum |weight| |sample| -> 3.4e-5 at
  K = 9 * 512 ("dcn_bf16"), plus half a bf16 ulp of |y| for a bf16 output (slack).
ROIAlign: fp32 arithmetic on exact inputs (bf16 values, or hi + lo of pairs): "roi_y" and its position slack as in
  tests/test_gpu_backward.py, plus half a bf16 ulp (bf16 output) or 2^-17 |y| (pair output) of storage.
Pair outputs are also checked for a normalised split: hi == bf16(hi + lo) and |lo| <= half an ulp of hi.
tests/test_grad_oracle_cpu.py shows that each DCN constant accepts an emulation of its mode's arithmetic and rejects a
corner guard off by one, a 1/64-px shift, a dropped lo*hi term, truncated bf16 samples, a mask applied to one of
hi / lo only, and the window kernel's in-window test one px too wide.

Measured on an NVIDIA H100 80GB HBM3 (SXM, power limit 700 W), worst err / bound over all cases: window kernel N = 32
and N = 128 and the gather kernel on pairs 4.6e-6, gather kernel bf16x3 on fp32 activations 2.9e-6, bf16 with fp32
output 6.4e-7 and with bf16 output 2.5e-7; 10x to 50x below the a-priori constants, so grad_oracle.TOL holds about 4x the
measured values (2e-5, 1.2e-5, 2.6e-6).  The ROIAlign errors stay inside their position and storage slack (ratio 0)."""
import os
import re
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import grad_oracle as G  # noqa: E402
from kernel_trace import launched_kernels  # noqa: E402

pytestmark = pytest.mark.gpu
X3, BF16 = 1, 2
WORST = {}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    yield torch.device("cuda", 0)
    print("\nworst |kernel - fp64| / bound:", {k: "%.3g (c %.2g)" % v for k, v in sorted(WORST.items())})
    import kernel_trace
    print("profiler sessions discarded for lost records so far:", kernel_trace.DISCARDED[0])


@pytest.fixture()
def engine():
    """Global engine switches, restored after every case."""
    import upsnet_b200 as U
    from upsnet_b200 import operators as ops
    from upsnet_b200._lib import lib
    was = dict(ops.DCN_WINDOW)
    try:
        yield U
    finally:
        assert lib().upsnet_dcn_set_tile_n(0) == 0
        ops.DCN_WINDOW.update(was)
        U.set_precision("fp32")


def _check(key, family, got, want, bound, slack=None):
    c = G.TOL[family]
    ok, ratio = G.check(got, want, bound, c, slack=slack)
    WORST[key] = (max(WORST.get(key, (0.0, c))[0], ratio), c)
    assert ok, (key, "worst err / bound %.3g > c = %g" % (ratio, c))


# ------------------------------------------------------------------------------------------------
# deformable convolution
# ------------------------------------------------------------------------------------------------
def _dcn(N, Cin, Cout, H, W, pd=1, frac=0.3, relu=False):
    return dict(N=N, Cin=Cin, Cout=Cout, H=H, W=W, pd=pd, frac=frac, relu=relu)


DCN_CASES = {
    "head256": _dcn(1, 256, 128, 32, 48),                          # semantic-head layer 0
    "cin64_odd_kblocks": _dcn(1, 64, 64, 16, 16, frac=1.0),        # 9 k-blocks
    "ragged_relu": _dcn(2, 128, 128, 25, 42, relu=True),           # config B 25 x 42, batch 2, ReLU epilogue
    "dil2_cout16": _dcn(1, 64, 16, 20, 20, pd=2, frac=1.0),        # dilation 2, Cout padded to 32
    "cin512": _dcn(1, 512, 512, 13, 21),                           # four N tiles of 128, K = 4608
    "below_one_tile": _dcn(1, 64, 64, 6, 5, frac=1.0),             # map smaller than one tile
    "many_tiles": _dcn(3, 64, 128, 64, 96),                        # > 132 tiles: CTAs run several
    "cin256_cout256": _dcn(1, 256, 256, 24, 40, frac=1.0),         # two N tiles of 128
}
# path: (tolerance family, kernel that must run, output storage)
PATHS = {
    "window_n32": ("dcn_x3_pair", r"dcn_win_kernel<32>", "pair"),
    "window_n128": ("dcn_x3_pair", r"dcn_win_kernel<128>", "pair"),
    "gather_pair": ("dcn_x3_pair", r"igemm_tc_kernel<1, ?2\b", "pair"),
    "gather_x3_fp32": ("dcn_x3_f32", r"igemm_tc_kernel<1, ?0\b", "f32"),
    "gather_bf16_fp32out": ("dcn_bf16", r"igemm_tc_kernel<1, ?1\b", "f32"),
    "gather_bf16_bf16out": ("dcn_bf16", r"igemm_tc_kernel<1, ?1\b", "bf16"),
}


def _conv_kernels(fn):
    """fn() under torch.profiler: its result and the convolution kernels it launched, weight packing excluded
    (tests/kernel_trace.py: sessions that lost their records are repeated)."""
    return launched_kernels(fn, lambda n: ("igemm" in n or "dcn" in n) and "pack" not in n)


def _window_tile(N, Ho, Wo, Cout, bn):
    """The pixel tile upsnet_dcn_pair_forward picks for N tile bn (csrc/dcn_win.cu)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cp = 32 if Cout <= 32 else (Cout + 63) // 64 * 64

    def tiles(tw, th, b):
        return N * -(-Wo // tw) * -(-Ho // th) * (cp // b)
    if bn == 128:
        assert cp % 128 == 0
        return 16, 8
    tw, th = 16, 8
    if tiles(tw, th, 32) < sms // 2:
        tw, th = 8, 8
    if tiles(tw, th, 32) < sms // 2:
        th = 4
    return tw, th


def _run_dcn(U, path, x, off, w, b, m, pd, relu):
    """The layer on one path; -> (logical NCHW float64 result, pair store or None, launched conv kernels)."""
    from upsnet_b200 import operators as ops
    from upsnet_b200._lib import lib
    kw = dict(mask=m, relu=relu)
    if path in ("window_n32", "window_n128", "gather_pair"):
        U.set_precision("bf16x3")
        ops.DCN_WINDOW.update(on=path != "gather_pair", min_pixels=0)
        assert lib().upsnet_dcn_set_tile_n({"window_n32": 32, "window_n128": 128}.get(path, 0)) == 0
        xp = ops.Pair.from_float(x)
        y, names = _conv_kernels(lambda: U.deform_conv(xp, off, w, b, 1, pd, pd, 1, precision=X3, **kw))
        assert isinstance(y, ops.Pair)
        return y.float().double(), y.store, names
    U.set_precision("fp32")
    if path == "gather_x3_fp32":
        y, names = _conv_kernels(lambda: U.deform_conv(x.contiguous(memory_format=torch.channels_last), off, w, b, 1, pd,
                                                       pd, 1, precision=X3, **kw))
        assert y.dtype == torch.float32
    else:
        od = torch.bfloat16 if path == "gather_bf16_bf16out" else torch.float32
        xb = x.bfloat16().contiguous(memory_format=torch.channels_last)
        y, names = _conv_kernels(lambda: U.deform_conv(xb, off, w, b, 1, pd, pd, 1, precision=BF16, out_dtype=od, **kw))
        assert y.dtype == od
    return y.double(), None, names


def _dcn_inputs(c, seed, dev):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(c["N"], c["Cin"], c["H"], c["W"], generator=g).to(dev)
    w = (torch.randn(c["Cout"], c["Cin"], 3, 3, generator=g) / (c["Cin"] * 9) ** 0.5).to(dev)
    b = torch.randn(c["Cout"], generator=g).to(dev)
    m = (torch.rand(c["N"], 9, c["H"], c["W"], generator=g) * 2).to(dev)
    # activations whose pair split is exact (x == hi + lo), so fp32 and pair paths share one reference
    from upsnet_b200 import operators as ops
    return ops.Pair.from_float(x).float().contiguous(), w, b, m


def _dcn_paths(U, c, off, x, w, b, m, paths):
    pd, relu = c["pd"], c["relu"]
    off64, m64 = off.double(), None if m is None else m.double()
    refs = {}
    for path in paths:
        family, kernel, out = PATHS[path]
        if family == "dcn_bf16":
            wb, xb = w.bfloat16().float(), x.bfloat16().float()
            if "bf16" not in refs:
                col = G.dcn_columns(xb, off, 3, 3, 1, pd, pd, mask=m, mode="bf16")
                refs["bf16"] = (G.dcn_gemm(col, wb, b, "bf16", dtype=torch.float64),
                                G.dcn_gemm(col.abs(), wb.abs(), b.abs(), "bf16", dtype=torch.float64))
            want, bound = refs["bf16"]
            got, store, names = _run_dcn(U, path, xb, off, wb, b, m, pd, relu)
        else:
            if "x3" not in refs:
                refs["x3"] = (G.deform_conv(x.double(), off64, w.double(), b.double(), m64, 1, pd, pd, offset32=off),
                              G.deform_conv(x.double().abs(), off64, w.double().abs(), b.double().abs(), m64, 1, pd, pd,
                                            offset32=off))
            want, bound = refs["x3"]
            got, store, names = _run_dcn(U, path, x, off, w, b, m, pd, relu)
        assert len(names) == 1 and re.search(kernel, next(iter(names))), (path, names)
        if relu:
            want = want.clamp_min(0)
        top = want.abs() + G.TOL[family] * bound                 # largest magnitude of the kernel's fp32 result
        slack = {"pair": 2.0 ** -17 * top, "bf16": G.half_ulp_bf16(top), "f32": None}[out]
        assert got.shape == want.shape
        _check(path, family, got, want, bound, slack)
        if store is not None:
            G.check_pair_split(store)


def _all_paths(c):
    wide = c["Cout"] % 128 == 0
    return [p for p in PATHS if p != "window_n128" or wide]


@pytest.mark.parametrize("modulated", [False, True])
@pytest.mark.parametrize("name", list(DCN_CASES))
def test_dcn_forward_vs_fp64(dev, engine, name, modulated):
    """Every tensor-core DCN path on special_offsets (share `frac` of the coordinates on the decision points)."""
    c = DCN_CASES[name]
    x, w, b, m = _dcn_inputs(c, list(DCN_CASES).index(name), dev)
    off = G.special_offsets(c["N"], 3, 3, c["H"], c["W"], c["H"], c["W"], 1, c["pd"], c["pd"], len(name), c["frac"]).to(dev)
    _dcn_paths(engine, c, off, x, w, b, m if modulated else None, _all_paths(c))


@pytest.mark.parametrize("modulated", [False, True])
@pytest.mark.parametrize("name", list(DCN_CASES))
def test_dcn_window_geometry_vs_fp64(dev, engine, name, modulated):
    """The window kernel, both N tiles, on window-mode offsets built for the pixel tile that N tile runs with: corner
    boxes of the window's size and one px either side, samples on the last row / column of a mean-centred window."""
    c = DCN_CASES[name]
    x, w, b, m = _dcn_inputs(c, 100 + list(DCN_CASES).index(name), dev)
    for path in [p for p in _all_paths(c) if p.startswith("window")]:
        tile = _window_tile(c["N"], c["H"], c["W"], c["Cout"], 128 if path == "window_n128" else 32)
        off = G.special_offsets(c["N"], 3, 3, c["H"], c["W"], c["H"], c["W"], 1, c["pd"], c["pd"], len(name), c["frac"],
                                window=tile).to(dev)
        _dcn_paths(engine, c, off, x, w, b, m if modulated else None, [path])


# ------------------------------------------------------------------------------------------------
# ROIAlign
# ------------------------------------------------------------------------------------------------
def _roi_c_abi(feat_store, B, C, H, W, layout, dtype, rois, PH, PW, scale, sr, out):
    from upsnet_b200._lib import check, lib, ptr, stream_ptr
    check(lib().upsnet_roi_align_forward(ptr(feat_store), B, C, H, W, layout, dtype, ptr(rois), rois.shape[0], PH, PW, sr,
                                         float(scale), ptr(out), stream_ptr(out.device)), "roi_align")
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("sr", [1, 2, 4])
@pytest.mark.parametrize("pooled", [(7, 7), (14, 14), (3, 5)])
def test_roi_align_layouts_vs_fp64(dev, pooled, sr):
    """NHWC fp32, NHWC bf16, pair and flat pair on the hand-placed rois (outside the map, zero width on the last row /
    column, smaller than a pixel, the whole map) and random ones, one map level."""
    from upsnet_b200 import _lib
    from upsnet_b200 import operators as ops
    PH, PW = pooled
    B, C, H, W, scale = 2, 24, 30, 44, 0.25
    g = torch.Generator().manual_seed(100 * PH + sr)
    feat = ops.Pair.from_float(torch.randn(B, C, H, W, generator=g).to(dev))
    fx = feat.float().contiguous()                                        # hi + lo, exact
    fb = fx.bfloat16().float()
    rois = G.hand_rois(H, W, scale, 25, sr).to(dev)
    R = rois.shape[0]
    refs = {}
    for name, f in (("x", fx), ("b", fb)):
        y64 = G.roi_align(f.double(), rois, PH, PW, scale, sr)
        bd = G.roi_align_bounds(f.double(), rois, PH, PW, scale, sr, torch.zeros_like(y64))
        refs[name] = (y64, bd["y"], bd["y_slack"], y64.abs() + G.TOL["roi_y"] * bd["y"])
    y64, bound, slack, top = refs["x"]
    got = ops.roi_align(fx.permute(0, 2, 3, 1).contiguous(), rois, PH, PW, scale, sr, layout="nhwc")
    _check("roi nhwc fp32", "roi_y", got.permute(0, 3, 1, 2).double(), y64, bound, slack)
    out = torch.empty(R, PH, PW, C, dtype=torch.bfloat16, device=dev)
    _roi_c_abi(fb.bfloat16().permute(0, 2, 3, 1).contiguous(), B, C, H, W, _lib.LAYOUT_NHWC, _lib.DTYPE_BF16, rois, PH,
               PW, scale, sr, out)
    yb, bb, sb, tb = refs["b"]
    _check("roi nhwc bf16", "roi_y", out.permute(0, 3, 1, 2).double(), yb, bb, sb + G.half_ulp_bf16(tb))
    if PH * PW * sr * sr > 1024:           # beyond the pair kernel's per-roi sample table
        return
    out = torch.empty(R, PH, PW, 2 * C, dtype=torch.bfloat16, device=dev)
    _roi_c_abi(feat.store, B, C, H, W, _lib.LAYOUT_NHWC, _lib.DTYPE_PAIR, rois, PH, PW, scale, sr, out)
    G.check_pair_split(out)
    _check("roi pair", "roi_y", ops.Pair(out).float().double(), y64, bound, slack + 2.0 ** -17 * top)
    out = torch.empty(R, 1, 1, 2 * PH * PW * C, dtype=torch.bfloat16, device=dev)
    _roi_c_abi(feat.store, B, C, H, W, _lib.LAYOUT_FLAT_PAIR, _lib.DTYPE_PAIR, rois, PH, PW, scale, sr, out)
    G.check_pair_split(out)
    flat = ops.Pair(out).float().double().reshape(R, PH, PW, C).permute(0, 3, 1, 2)
    _check("roi flat pair", "roi_y", flat, y64, bound, slack + 2.0 ** -17 * top)


SCALES = [1 / 4., 1 / 8., 1 / 16., 1 / 32.]


@pytest.mark.parametrize("flat", [False, True])
@pytest.mark.parametrize("sr", [1, 2, 4])
def test_fpn_roi_align_pair_roi_count_vs_fp64(dev, sr, flat):
    """FPN ROIAlign on pair features in one launch with a device-side roi count n_dev < R: rois whose level sits exactly
    on an FPN boundary (sides 112, 224, 448) and one px below it, on all four levels; the rows >= n_dev keep the sentinel
    they were filled with, bit for bit."""
    from upsnet_b200 import _lib
    from upsnet_b200 import operators as ops
    from upsnet_b200._lib import check, lib, ptr, stream_ptr
    import ctypes as C
    PH = PW = 7
    g = torch.Generator().manual_seed(sr)
    feats = [ops.Pair.from_float(torch.randn(2, 16, 128 >> l, 176 >> l, generator=g).to(dev)) for l in range(4)]
    rng = np.random.default_rng(sr)
    rows = []
    for i, s in enumerate([40, 111, 112, 160, 223, 224, 300, 447, 448, 520] * 2):
        x0, y0 = float(rng.integers(-20, 704 - s)), float(rng.integers(-20, 512 - s))
        rows.append([i % 2, x0, y0, x0 + s - 1, y0 + s - 1])
    rois = torch.tensor(rows, dtype=torch.float32, device=dev)
    R, n = rois.shape[0], rois.shape[0] - 6
    lv = G.fpn_levels(rois)
    assert set(lv[:n].tolist()) == {0, 1, 2, 3} and lv[[1, 2, 4, 5, 7, 8]].tolist() == [0, 1, 1, 2, 2, 3]
    n_dev = torch.tensor([n], dtype=torch.int32, device=dev)
    Cc = 16
    shape = (R, 1, 1, 2 * PH * PW * Cc) if flat else (R, PH, PW, 2 * Cc)
    out = torch.full(shape, -7.25, dtype=torch.bfloat16, device=dev)
    fp = (C.c_void_p * 4)(*[f.store.data_ptr() for f in feats])
    hs = (C.c_int * 4)(*[f.shape[2] for f in feats]); ws = (C.c_int * 4)(*[f.shape[3] for f in feats])
    sc = (C.c_float * 4)(*SCALES)
    check(lib().upsnet_roi_align_fpn_forward(fp, hs, ws, sc, 2, Cc, _lib.LAYOUT_FLAT_PAIR if flat else _lib.LAYOUT_NHWC,
                                             _lib.DTYPE_PAIR, ptr(rois), R, PH, PW, sr, ptr(out), ptr(None), ptr(n_dev),
                                             stream_ptr(dev)), "fpn_roi_align")
    torch.cuda.synchronize()
    assert bool((out[n:] == -7.25).all()), "rows at or above n_dev were written"
    fx = [f.float().contiguous().double() for f in feats]
    y64 = G.fpn_roi_align(fx, rois[:n], PH, PW, SCALES, sr)
    bd = G.fpn_roi_align_bounds(fx, rois[:n], PH, PW, SCALES, sr, torch.zeros_like(y64))
    top = y64.abs() + G.TOL["roi_y"] * bd["y"]
    G.check_pair_split(out[:n])
    got = ops.Pair(out[:n].contiguous()).float().double()
    got = got.reshape(n, PH, PW, Cc).permute(0, 3, 1, 2) if flat else got
    _check("roi fpn pair n_dev" + (" flat" if flat else ""), "roi_y", got, y64, bd["y"], bd["y_slack"] + 2.0 ** -17 * top)
