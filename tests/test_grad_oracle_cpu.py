"""The float64 restatement of the training operators (tests/grad_oracle.py) that the GPU backward tests compare against:
agreement with torchvision's independent CPU implementations of the same operators in float64, finite differences, and
the sensitivity of the GPU tolerance (it accepts an fp32 evaluation of the operator and rejects near misses)."""
import os
import sys

import numpy as np
import pytest
import torch
import torchvision

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import grad_oracle as G  # noqa: E402

DCN_CASES = [  # (N, Cin, Cout, H, W, kh, kw, stride, padding, dilation)
    (2, 3, 4, 7, 9, 3, 3, 1, 1, 1),
    (1, 2, 3, 9, 8, 3, 3, (2, 1), (1, 2), 1),
    (1, 3, 2, 10, 11, 3, 3, 2, 2, 2),
    (2, 2, 3, 6, 7, 1, 3, 1, (0, 1), 1),
]


def _dcn_inputs(case, modulated, seed, frac=0.5):
    N, Cin, Cout, H, W, kh, kw, s, p, d = case
    g = torch.Generator().manual_seed(seed)
    (sh, sw), (ph, pw), (dh, dw) = G._pair(s), G._pair(p), G._pair(d)
    Ho, Wo = (H + 2 * ph - dh * (kh - 1) - 1) // sh + 1, (W + 2 * pw - dw * (kw - 1) - 1) // sw + 1
    x = torch.randn(N, Cin, H, W, generator=g, dtype=torch.float64)
    off = G.special_offsets(N, kh, kw, Ho, Wo, H, W, s, p, d, seed, frac).double()
    w = torch.randn(Cout, Cin, kh, kw, generator=g, dtype=torch.float64) * 0.3
    b = torch.randn(Cout, generator=g, dtype=torch.float64)
    m = torch.rand(N, kh * kw, Ho, Wo, generator=g, dtype=torch.float64) * 2 if modulated else None
    dy = torch.randn(N, Cout, Ho, Wo, generator=g, dtype=torch.float64)
    return x, off, w, b, m, dy


def _grads(fn, inputs, dy):
    ins = [None if t is None else t.detach().clone().requires_grad_(True) for t in inputs]
    y = fn(*ins)
    gs = torch.autograd.grad(y, [t for t in ins if t is not None], dy)
    return y.detach(), list(gs)


@pytest.mark.parametrize("modulated", [False, True])
@pytest.mark.parametrize("case", DCN_CASES)
def test_deform_conv_matches_torchvision_fp64(case, modulated):
    s, p, d = case[7:]
    x, off, w, b, m, dy = _dcn_inputs(case, modulated, 1)

    def ours(x_, o_, w_, b_, m_=None):
        return G.deform_conv(x_, o_, w_, b_, m_, s, p, d)

    def tv(x_, o_, w_, b_, m_=None):
        return torchvision.ops.deform_conv2d(x_, o_, w_, b_, stride=s, padding=p, dilation=d, mask=m_)

    ya, ga = _grads(ours, (x, off, w, b, m), dy)
    yb, gb = _grads(tv, (x, off, w, b, m), dy)
    # A sample exactly on h = -1 or w = -1 contributes nothing, and the reference's coordinate gradient is zero there
    # (deform_conv_kernel.cu: inv_h <= -1 -> no weight); torchvision returns the one-sided derivative from inside.
    N, _, H, W = x.shape
    kh, kw = case[5:7]
    Ho, Wo = off.shape[2:]
    pos = off.view(N, kh * kw, 2, Ho, Wo) + torch.stack(
        [(torch.arange(Ho).view(1, -1, 1) * G._pair(s)[0] - G._pair(p)[0] + (torch.arange(kh * kw) // kw).view(-1, 1, 1) * G._pair(d)[0]).expand(-1, -1, Wo),
         (torch.arange(Wo).view(1, 1, -1) * G._pair(s)[1] - G._pair(p)[1] + (torch.arange(kh * kw) % kw).view(-1, 1, 1) * G._pair(d)[1]).expand(-1, Ho, -1)], 1)
    on_minus_one = (pos == -1).any(2, keepdim=True).expand(-1, -1, 2, -1, -1).reshape_as(off)
    assert int(on_minus_one.sum()) > 0 and float(ga[1][on_minus_one].abs().max()) == 0.0
    gb[1] = torch.where(on_minus_one, 0.0, gb[1])
    for name, a, r in zip(["y", "dx", "doffset", "dweight", "dbias", "dmask"], [ya] + ga, [yb] + gb):
        assert (a - r).abs().max() <= 1e-10 * max(1.0, float(r.abs().max())), name


@pytest.mark.parametrize("sr", [0, 1, 2, 4])
@pytest.mark.parametrize("pooled", [(7, 7), (3, 5)])
def test_roi_align_matches_torchvision_fp64(sr, pooled):
    g = torch.Generator().manual_seed(2)
    feat = torch.randn(2, 3, 13, 17, generator=g, dtype=torch.float64)
    rois = torch.tensor([[0, 3.3, 5.1, 40.2, 30.7], [1, -20, -10, 30, 25], [1, 60, 40, 90, 70], [0, 52, 40, 68, 52],
                         [0, 10.2, 10.4, 10.5, 10.6], [1, 0, 0, 67, 51], [0, -100, -100, -60, -50], [1, 20, 8, 44.5, 31]],
                        dtype=torch.float64)
    dy = torch.randn(rois.shape[0], 3, *pooled, generator=g, dtype=torch.float64)
    ya, (ga,) = _grads(lambda f: G.roi_align(f, rois, *pooled, 0.25, sr, fp32_positions=False), (feat,), dy)
    yb, (gb,) = _grads(lambda f: torchvision.ops.roi_align(f, rois, pooled, 0.25, sr, False), (feat,), dy)
    assert (ya - yb).abs().max() <= 1e-10 * float(yb.abs().max())
    assert (ga - gb).abs().max() <= 1e-10 * float(gb.abs().max())


def test_fpn_levels_rule():
    # w = h = 112 is the first roi on level 1 (sqrt(wh)/224 + 1e-6 >= 0.5), 224 on level 2, 448 on level 3
    rois = torch.tensor([[0, 0, 0, s - 1, s - 1] for s in (8, 111, 112, 223, 224, 447, 448, 2000)], dtype=torch.float32)
    assert G.fpn_levels(rois).tolist() == [0, 0, 1, 1, 2, 2, 3, 3]


def test_deform_conv_gradcheck():
    g = torch.Generator().manual_seed(5)
    x = torch.randn(1, 2, 5, 6, generator=g, dtype=torch.float64, requires_grad=True)
    off = (torch.randn(1, 18, 5, 6, generator=g, dtype=torch.float64) * 1.3).requires_grad_(True)
    w = torch.randn(2, 2, 3, 3, generator=g, dtype=torch.float64, requires_grad=True)
    b = torch.randn(2, generator=g, dtype=torch.float64, requires_grad=True)
    m = torch.rand(1, 9, 5, 6, generator=g, dtype=torch.float64, requires_grad=True)
    # finite differences need every sample away from the kinks at integer positions (the bases are integers)
    assert float((off - off.round()).abs().min()) > 1e-4
    assert torch.autograd.gradcheck(lambda *a: G.deform_conv(*a, stride=1, padding=1, fp32_positions=False),
                                    (x, off, w, b, m), eps=1e-6, atol=1e-6)


def test_roi_align_gradcheck():
    g = torch.Generator().manual_seed(6)
    feat = torch.randn(1, 2, 6, 7, generator=g, dtype=torch.float64, requires_grad=True)
    rois = torch.tensor([[0, 1.3, 2.1, 20.7, 17.2], [0, -6, -3, 9.5, 12.25]])
    assert torch.autograd.gradcheck(lambda f: G.roi_align(f, rois, 3, 2, 0.25, 2), (feat,), eps=1e-6, atol=1e-6)


def _dcn_families(case, modulated, xs, off, w, b, m, dy, **variant):
    s, p, d = case[7:]
    dt = xs.dtype
    ins = [t.detach().to(dt).requires_grad_(True) if t is not None else None for t in (xs, off, w, b, m)]
    y = G.deform_conv(*ins[:4], ins[4], s, p, d, offset32=off.float(), **variant)
    gs = torch.autograd.grad(y, [t for t in ins if t is not None], dy.to(dt))
    return dict(zip(["dcn_y", "dcn_dx", "dcn_doffset", "dcn_dweight", "dcn_dbias", "dcn_dmask"], (y,) + gs))


@pytest.mark.parametrize("modulated", [False, True])
@pytest.mark.parametrize("case", DCN_CASES[:3])
def test_dcn_tolerance_accepts_fp32_rejects_near_miss(case, modulated):
    s, p, d = case[7:]
    x, off, w, b, m, dy = _dcn_inputs(case, modulated, 7, frac=0.7)
    x, w, b, m = (None if t is None else t.float().double() for t in (x, w, b, m))
    ref = _dcn_families(case, modulated, x, off, w, b, m, dy)
    bd = G.deform_conv_bounds(x, off, w, b, m, dy, s, p, d)
    keys = {"dcn_y": "y", "dcn_dx": "x", "dcn_doffset": "offset", "dcn_dweight": "weight", "dcn_dbias": "bias",
            "dcn_dmask": "mask"}

    def passes(got):
        return all(G.check(got[k], ref[k], bd[keys[k]], G.TOL[k])[0] for k in ref)

    assert passes(_dcn_families(case, modulated, x.float(), off, w, b, m, dy))
    assert not passes(_dcn_families(case, modulated, x, off, w, b, m, dy, right_guard=1))
    assert not passes(_dcn_families(case, modulated, x, off, w, b, m, dy, shift=1 / 64))


FWD_CASES = [  # (N, Cin, Cout, H, W, padding / dilation, special_offsets frac, window tile)
    (1, 8, 4, 40, 72, 1, 0.3, (16, 8)),        # window-mode offsets on 16 x 8 tiles (3 x 9 tiles of the three modes)
    (2, 4, 3, 11, 13, 1, 1.0, None),
    (1, 6, 5, 24, 20, 2, 0.3, (8, 4)),         # dilation 2, window mode on the small-map 8 x 4 tiles
]
FWD_FAULTS = {  # every fault each family's constant must reject
    "x3_pair": ["right_guard", "shift", "drop_lohi", "mask_hi_only", "window_edge"],
    "x3_f32": ["right_guard", "shift", "drop_lohi", "mask_hi_only"],
    "bf16": ["right_guard", "shift", "truncate"],       # one bf16 plane: no hi / lo to mask apart
}


def _fwd_inputs(case, modulated, seed):
    N, Cin, Cout, H, W, pd, frac, tile = case
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, Cin, H, W, generator=g)
    off = G.special_offsets(N, 3, 3, H, W, H, W, 1, pd, pd, seed, frac, window=tile)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / (Cin * 9) ** 0.5
    b = torch.randn(Cout, generator=g)
    m = torch.rand(N, 9, H, W, generator=g) * 2 if modulated else None
    return x, off, w, b, m


@pytest.mark.parametrize("modulated", [False, True])
@pytest.mark.parametrize("case", FWD_CASES)
@pytest.mark.parametrize("family", list(FWD_FAULTS))
def test_forward_tolerance_accepts_kernel_arithmetic_rejects_faults(family, case, modulated):
    """Each inference DCN precision mode (tests/test_gpu_forward_fp64.py) emulated in torch -- the gather's blend, the
    bf16 hi/lo split of sample and weights, three products (bf16x3) or one (bf16), fp32 accumulation -- passes its
    family's constant against the float64 reference, and each planted fault fails it.  Cases are narrowed to a few input
    channels: the faults that change a sample by 2^-9 of itself (drop_lohi, mask_hi_only) are diluted by averaging over
    the 9 Cin terms of an output, so with hundreds of channels their per-element ratio drops towards the constants.
    The window-edge fault changes only samples one px past the window, which window-mode offsets place; without them
    (case 2) it cannot be seen and is not asserted."""
    x, off, w, b, m = _fwd_inputs(case, modulated, 17)
    pd, tile = case[5], case[7]
    cfg = (3, 3, 1, pd, pd)
    if family == "x3_pair":
        hi = x.bfloat16().float()
        xin = (hi, (x - hi).bfloat16().float())
        xexact = xin[0].double() + xin[1].double()
    else:
        xin = x.bfloat16().float() if family == "bf16" else x
        xexact = xin.double()
    if family == "bf16":
        w = w.bfloat16().float()
        col = G.dcn_columns(xin, off, *cfg, mask=m, mode="bf16")
        want = G.dcn_gemm(col, w, b, "bf16", dtype=torch.float64)
        bound = G.dcn_gemm(col.abs(), w.abs(), b.abs(), "bf16", dtype=torch.float64)
    else:
        want = G.deform_conv(xexact, off.double(), w.double(), b.double(), None if m is None else m.double(), 1, pd, pd,
                             offset32=off)
        bound = G.deform_conv(xexact.abs(), off.double(), w.double().abs(), b.double().abs(),
                              None if m is None else m.double(), 1, pd, pd, offset32=off)
    c = G.TOL["dcn_" + family]

    def run(fault=None):
        col = G.dcn_columns(xin, off, *cfg, mask=m, mode=family, fault=fault, window=tile)
        return G.dcn_gemm(col, w, b, family, fault=fault)

    ok, ratio = G.check(run(), want, bound, c)
    assert ok, (family, "emulation rejected", ratio, c)
    for fault in FWD_FAULTS[family]:
        if (fault == "mask_hi_only" and m is None) or (fault == "window_edge" and tile is None):
            continue
        ok, ratio = G.check(run(fault), want, bound, c)
        assert not ok, (family, fault, "accepted", ratio, c)


def test_window_offsets_hit_the_window_geometry():
    """special_offsets(window=tile) produces, for dcn_win.cu's window placement: corner boxes 1 px narrower than,
    exactly as wide as and 1 px wider than the window in both axes; integer and fractional samples on the last column
    and row of a mean-centred window, and samples just before its first column and row."""
    H, W, Ho, Wo, K = 40, 72, 40, 72, 9
    off = G.special_offsets(1, 3, 3, Ho, Wo, H, W, 1, 1, 1, 4, 0.3, window=(16, 8))
    assert torch.equal(off, G.special_offsets(1, 3, 3, Ho, Wo, H, W, 1, 1, 1, 4, 0.3, window=(16, 8)))
    o = off.double().numpy().reshape(1, K, 2, Ho, Wo)
    bh = (np.arange(Ho)[None, :, None] - 1 + (np.arange(K) // 3)[:, None, None]) * np.ones((1, 1, Wo))
    bw = (np.arange(Wo)[None, None, :] - 1 + (np.arange(K) % 3)[:, None, None]) * np.ones((1, Ho, 1))
    h, w = bh + o[:, :, 0], bw + o[:, :, 1]
    ox, oy, hl, wl, valid = G.window_origins(h, w, H, W, (16, 8))
    spans_w, spans_h = set(), set()
    for n, ys, xs in G._tiles(1, Ho, Wo, (16, 8)):
        v = valid[n, :, ys, xs]
        spans_w.add(int(wl[n, :, ys, xs][v].max()) + 2 - int(wl[n, :, ys, xs][v].min()))
        spans_h.add(int(hl[n, :, ys, xs][v].max()) + 2 - int(hl[n, :, ys, xs][v].min()))
    assert {G.WIN_W - 1, G.WIN_W, G.WIN_W + 1} <= spans_w and {G.WIN_H - 1, G.WIN_H, G.WIN_H + 1} <= spans_h
    dx, dy = wl - ox, hl - oy
    integer_w, integer_h = w == np.floor(w), h == np.floor(h)
    for sel in (dx == G.WIN_W - 1) & integer_w, (dx == G.WIN_W - 1) & ~integer_w, (dy == G.WIN_H - 1) & integer_h, \
            (dy == G.WIN_H - 1) & ~integer_h, dx == -1, dy == -1:
        assert int((sel & valid).sum()) >= 3


@pytest.mark.parametrize("sr", [0, 2])
def test_roi_tolerance_accepts_fp32_rejects_near_miss(sr):
    g = torch.Generator().manual_seed(8)
    feat = torch.randn(2, 4, 15, 19, generator=g).double()
    rois = torch.tensor([[0, 3.3, 5.1, 40.2, 30.7], [1, -20, -10, 30, 25], [1, 60, 40, 75.5, 59.5], [0, 10.2, 10.4, 10.5, 10.6],
                         [1, 0, 0, 75, 59]])
    dy = torch.randn(rois.shape[0], 4, 7, 7, generator=g).double()
    bd = G.roi_align_bounds(feat, rois, 7, 7, 0.25, sr, dy)

    def fam(dt, shift=0.0):
        f = feat.to(dt).requires_grad_(True)
        y = G.roi_align(f, rois, 7, 7, 0.25, sr, shift=shift)
        (gf,) = torch.autograd.grad(y, f, dy.to(dt))
        return y, gf

    y64, g64 = fam(torch.float64)

    def passes(yg):
        return (G.check(yg[0], y64, bd["y"], G.TOL["roi_y"], slack=bd["y_slack"])[0] and
                G.check(yg[1], g64, bd["feat"], G.TOL["roi_dfeat"], slack=bd["feat_slack"])[0])

    assert passes(fam(torch.float32))
    assert not passes(fam(torch.float64, shift=1 / 64))
