"""Backward kernels of the custom operators (training configuration, csrc/backward.cu K1-K6, K8) and the training modules
built on them, against the float64 restatement of tests/grad_oracle.py run on the device.

Every output and gradient element is checked against its own bound: |kernel - fp64| <= c * (sum of |terms|) + 1e-6, with
c per gradient family in grad_oracle.TOL (tests/test_grad_oracle_cpu.py shows that c accepts an fp32 evaluation and
rejects a reference with one corner guard off by one or samples shifted by 1/64 px).  dx and d(feat) are accumulated with
atomics, so nothing here asserts bit equality between runs.  Run with -s to see the worst err / bound per family."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import grad_oracle as G  # noqa: E402

pytestmark = pytest.mark.gpu
WORST = {}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    yield torch.device("cuda", 0)
    print("\nworst |kernel - fp64| / bound:", {k: "%.3g (c %.0e)" % (v, G.TOL[k]) for k, v in sorted(WORST.items())})


def _check(family, got, want, bound, name="", slack=None):
    assert got is not None, (family, name, "no gradient")
    ok, ratio = G.check(got, want, bound, G.TOL[family], slack=slack)
    WORST[family] = max(WORST.get(family, 0.0), ratio)
    assert ok, (family, name, "worst err / bound %.3g > c = %g" % (ratio, G.TOL[family]))


def _ref_grads(fn, inputs, dy):
    """fp64 forward and gradients of fn w.r.t. every input that is not None."""
    ins = [None if t is None else t.detach().double().requires_grad_(True) for t in inputs]
    y = fn(*ins)
    used = [t for t in ins if t is not None]
    gs = torch.autograd.grad(y, used, dy.double(), allow_unused=True)
    it = iter(torch.zeros_like(t) if g_ is None else g_ for t, g_ in zip(used, gs))     # an FPN level without rois
    return y.detach(), [None if t is None else next(it) for t in ins]


# ------------------------------------------------------------------------------------------------
# DeformConvFunction / ModDeformConvFunction
# ------------------------------------------------------------------------------------------------
def _dcn(N, Cin, Cout, H, W, k=(3, 3), s=1, p=1, d=1, bias=True, frac=0.3):
    return dict(N=N, Cin=Cin, Cout=Cout, H=H, W=W, k=k, s=s, p=p, d=d, bias=bias, frac=frac)


DCN_CASES = {
    "small": _dcn(2, 8, 12, 14, 18),
    "cin64": _dcn(1, 64, 32, 20, 24),
    "s2p2d2": _dcn(1, 16, 16, 17, 19, s=2, p=2, d=2),
    "stride2": _dcn(1, 16, 8, 15, 17, s=2),
    "stride21": _dcn(1, 8, 8, 15, 17, s=(2, 1)),
    "p0d2": _dcn(1, 8, 8, 13, 16, p=0, d=2),
    "p1d2": _dcn(1, 8, 8, 13, 16, p=1, d=2),
    "pad12": _dcn(1, 8, 8, 13, 16, p=(1, 2)),
    "k1x3": _dcn(2, 8, 8, 11, 14, k=(1, 3), p=(0, 1)),
    "nobias_d2": _dcn(1, 16, 16, 14, 14, p=2, d=2, bias=False),
    "cin1": _dcn(1, 1, 5, 12, 13),
    "cin3": _dcn(1, 3, 7, 12, 13),
    "cin31": _dcn(1, 31, 9, 12, 13),
    "cin33": _dcn(1, 33, 3, 12, 13),
    "cin100": _dcn(1, 100, 17, 12, 13),
    "cin256": _dcn(1, 256, 11, 12, 13),
    "n3": _dcn(3, 12, 5, 10, 11, frac=0.6),
    "special": _dcn(2, 5, 6, 9, 10, frac=1.0),
    "grid_stride": _dcn(1, 256, 8, 64, 72, frac=0.1),     # im2col 1.18 M, col2im 10.6 M, coord 1.33 M threads > 1.08 M grid
}


@pytest.mark.parametrize("modulated", [False, True])
@pytest.mark.parametrize("name", list(DCN_CASES))
def test_deform_conv_function_vs_fp64(dev, name, modulated):
    from upsnet_b200.training import DeformConvFunction, ModDeformConvFunction
    c = DCN_CASES[name]
    g = torch.Generator().manual_seed(list(DCN_CASES).index(name))
    (kh, kw), (sh, sw), (ph, pw), (dh, dw) = c["k"], G._pair(c["s"]), G._pair(c["p"]), G._pair(c["d"])
    Ho, Wo = (c["H"] + 2 * ph - dh * (kh - 1) - 1) // sh + 1, (c["W"] + 2 * pw - dw * (kw - 1) - 1) // sw + 1
    x = torch.randn(c["N"], c["Cin"], c["H"], c["W"], generator=g).to(dev)
    off = G.special_offsets(c["N"], kh, kw, Ho, Wo, c["H"], c["W"], c["s"], c["p"], c["d"], len(name), c["frac"]).to(dev)
    w = (torch.randn(c["Cout"], c["Cin"], kh, kw, generator=g) / (c["Cin"] * kh * kw) ** 0.5).to(dev)
    b = torch.randn(c["Cout"], generator=g).to(dev) if c["bias"] else None
    m = (torch.rand(c["N"], kh * kw, Ho, Wo, generator=g) * 2).to(dev) if modulated else None
    dy = torch.randn(c["N"], c["Cout"], Ho, Wo, generator=g).to(dev)
    ins = [t.clone().requires_grad_(True) if t is not None else None for t in (x, off, m, w, b)]
    if modulated:
        y = ModDeformConvFunction.apply(ins[0], ins[1], ins[2], ins[3], ins[4], c["s"], c["p"], c["d"])
    else:
        y = DeformConvFunction.apply(ins[0], ins[1], ins[3], ins[4], c["s"], c["p"], c["d"])
    y.backward(dy)
    y64, g64 = _ref_grads(lambda x_, o_, m_, w_, b_: G.deform_conv(x_, o_, w_, b_, m_, c["s"], c["p"], c["d"]),
                          (x, off, m, w, b), dy)
    bd = G.deform_conv_bounds(x, off, w, b, m, dy, c["s"], c["p"], c["d"])
    _check("dcn_y", y, y64, bd["y"])
    for fam, key, t, r in (("dcn_dx", "x", ins[0], g64[0]), ("dcn_doffset", "offset", ins[1], g64[1]),
                           ("dcn_dmask", "mask", ins[2], g64[2]), ("dcn_dweight", "weight", ins[3], g64[3]),
                           ("dcn_dbias", "bias", ins[4], g64[4])):
        if t is not None:
            _check(fam, t.grad, r, bd[key], key)


# ------------------------------------------------------------------------------------------------
# RoIAlignFunction
# ------------------------------------------------------------------------------------------------
def _roi_case(dev, B, C, H, W, rois, PH, PW, scale, sr, seed, forward=None):
    """forward(features, rois): the call under test, RoIAlignFunction by default."""
    from upsnet_b200.training import RoIAlignFunction
    g = torch.Generator().manual_seed(seed)
    feat = torch.randn(B, C, H, W, generator=g).to(dev)
    rois = rois.to(dev)
    dy = torch.randn(rois.shape[0], C, PH, PW, generator=g).to(dev)
    fd = feat.clone().requires_grad_(True)
    y = forward(fd, rois) if forward else RoIAlignFunction.apply(fd, rois, PH, PW, scale, sr)
    y.backward(dy)
    y64, (g64,) = _ref_grads(lambda f: G.roi_align(f, rois, PH, PW, scale, sr), (feat,), dy)
    bd = G.roi_align_bounds(feat, rois, PH, PW, scale, sr, dy)
    _check("roi_y", y, y64, bd["y"], slack=bd["y_slack"])
    _check("roi_dfeat", fd.grad, g64, bd["feat"], slack=bd["feat_slack"])
    return fd.grad


def test_roi_align_backward_vs_fp64(dev):
    """The RoIAlign module (the reference's call path, sampling ratio 2): 25 random rois on both images, one partly
    outside the map."""
    import upsnet_b200 as U
    rng = np.random.default_rng(2)
    n = 25
    c = rng.uniform(0, 1, (n, 2)) * np.array([170, 115]); s = np.exp(rng.uniform(np.log(4), np.log(150), (n, 2)))
    rois = np.concatenate([rng.integers(0, 2, (n, 1)), c - s / 2, c + s / 2], 1).astype(np.float32)
    rois[0, 1:] = [-20, -10, 30, 25]
    _roi_case(dev, 2, 16, 30, 44, torch.from_numpy(rois), 7, 7, 0.25, 2, 4, forward=U.RoIAlign(7, 7, 0.25))


@pytest.mark.parametrize("sr", [0, 1, 2, 4])
@pytest.mark.parametrize("pooled", [(7, 7), (14, 14), (3, 5)])
def test_roi_align_function_vs_fp64(dev, pooled, sr):
    _roi_case(dev, 2, 16, 30, 44, G.hand_rois(30, 44, 0.25, 25, sr), *pooled, 0.25, sr, 4)


def test_roi_align_many_overlapping_rois(dev):
    """200 rois around one spot: heavy atomic contention on the same feature pixels."""
    rng = np.random.default_rng(9)
    c = 40 + rng.uniform(-3, 3, (200, 2)); s = rng.uniform(8, 24, (200, 2))
    rois = torch.tensor(np.concatenate([np.zeros((200, 1)), c - s / 2, c + s / 2], 1), dtype=torch.float32)
    _roi_case(dev, 1, 8, 24, 24, rois, 7, 7, 0.5, 2, 10)


def test_roi_align_no_rois_zero_gradient(dev):
    grad = _roi_case(dev, 2, 4, 9, 11, torch.zeros(0, 5), 7, 7, 0.25, 2, 11)
    assert grad.shape == (2, 4, 9, 11) and not bool(grad.any())


def test_roi_align_grid_stride(dev):
    """R * C * 14 * 14 = 1.6 M output elements, above the 1.08 M threads of the capped grid."""
    _roi_case(dev, 2, 64, 40, 56, G.hand_rois(40, 56, 0.25, 117, 12), 14, 14, 0.25, 2, 12)


# ------------------------------------------------------------------------------------------------
# modules: DeformConvWithOffset, ModDeformConvWithOffsetMask, FPNRoIAlign, deformable_groups > 1
# ------------------------------------------------------------------------------------------------
def _conv_abs_grads(x, weight, upstream_bound):
    """Bounds of the offset conv's d(x), d(weight), d(bias) from a bound on its output gradient."""
    xa, wa = x.detach().double().abs(), weight.detach().double().abs()
    return (torch.nn.grad.conv2d_input(xa.shape, wa, upstream_bound, padding=1),
            torch.nn.grad.conv2d_weight(xa, wa.shape, upstream_bound, padding=1), upstream_bound.sum((0, 2, 3)))


@pytest.mark.parametrize("modulated", [False, True])
@pytest.mark.parametrize("zero_init", [False, True])
def test_with_offset_modules_all_parameters_get_fp64_gradients(dev, modulated, zero_init):
    import upsnet_b200 as U
    from upsnet_b200 import operators as ops
    torch.manual_seed(13)
    Cin, Cout, H, W = 24, 16, 13, 17
    m = (U.ModDeformConvWithOffsetMask if modulated else U.DeformConvWithOffset)(Cin, Cout, 3, padding=1).to(dev)
    oc = m.conv_offset_mask if modulated else m.conv_offset
    if not zero_init:
        oc.weight.data.normal_(0, 0.3); oc.bias.data.normal_(0, 0.5)
    x = torch.randn(1, Cin, H, W, device=dev, requires_grad=True)
    dy = torch.randn(1, Cout, H, W, device=dev)
    m(x).backward(dy)
    params = [x, oc.weight, oc.bias, m.conv.weight, m.conv.bias]
    assert all(p.grad is not None for p in params)
    if zero_init:     # the reference's initialisation: offsets start at zero, but they must still learn
        assert bool(oc.weight.grad.any()) and bool(oc.bias.grad.any())
    with torch.no_grad():
        om32 = ops.conv2d(x, oc.weight, oc.bias, 1, 1, 1, out_format="nchw")     # the offsets the module sampled at
    off32 = torch.cat(torch.chunk(om32, 3, 1)[:2], 1) if modulated else om32
    with torch.enable_grad():
        xs, ow, ob, cw, cb = (p.detach().double().requires_grad_(True) for p in params)
        om = torch.nn.functional.conv2d(xs, ow, ob, padding=1)
        if modulated:
            o1, o2, mk = torch.chunk(om, 3, 1)
            off, mask = torch.cat((o1, o2), 1), torch.sigmoid(mk) * 2
            mask.retain_grad()
        else:
            off, mask = om, None
        off.retain_grad()
        y64 = G.deform_conv(xs, off, cw, cb, mask, 1, 1, 1, offset32=off32)
        y64.backward(dy.double())
    bd = G.deform_conv_bounds(x, off.detach(), m.conv.weight, m.conv.bias, mask, dy, 1, 1, 1)
    # the offset conv sees d(offset) (and d(mask) * 2 sigmoid') within c * bound of fp64; propagate that bound through it
    up = bd["offset"] + off.grad.abs()
    if modulated:
        s = torch.sigmoid(mk.detach())
        up = torch.cat((up, (bd["mask"] + mask.grad.abs()) * 2 * s * (1 - s)), 1)
    cx, cwb, cbb = _conv_abs_grads(x, oc.weight, up)
    _check("dcn_y", m(x).detach(), y64, bd["y"], "y")
    _check("dcn_dx", x.grad, xs.grad, bd["x"] + cx, "x")
    _check("dcn_dweight", oc.weight.grad, ow.grad, cwb, "offset conv weight")
    _check("dcn_dbias", oc.bias.grad, ob.grad, cbb, "offset conv bias")
    _check("dcn_dweight", m.conv.weight.grad, cw.grad, bd["weight"], "conv weight")
    _check("dcn_dbias", m.conv.bias.grad, cb.grad, bd["bias"], "conv bias")


SCALES = [1 / 4., 1 / 8., 1 / 16., 1 / 32.]


def _fpn_rois(all_levels):
    # sides 111 / 112, 223 / 224, 447 / 448 sit on both sides of the level boundaries (sqrt(wh) / 224 = 0.5, 1, 2)
    sides = [30, 111, 112, 160] + ([223, 224, 300, 447] if all_levels else []) + [448, 500]
    rng = np.random.default_rng(14 + all_levels)
    rows = []
    for i, s in enumerate(sides * 2):
        x0, y0 = rng.uniform(-20, 700 - s), rng.uniform(-20, 500 - s)
        rows.append([i % 2, x0, y0, x0 + s - 1, y0 + s - 1])
    return torch.tensor(rows, dtype=torch.float32)


@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("all_levels", [True, False])
def test_fpn_roi_align_module_gradients_per_level(dev, channels_last, all_levels):
    import upsnet_b200 as U
    g = torch.Generator().manual_seed(15)
    feats = [torch.randn(2, 8, 128 // 2 ** l, 176 // 2 ** l, generator=g).to(dev) for l in range(4)]
    if channels_last:
        feats = [f.contiguous(memory_format=torch.channels_last) for f in feats]
    rois = _fpn_rois(all_levels).to(dev)
    lv = G.fpn_levels(rois)
    assert set(lv.tolist()) == ({0, 1, 2, 3} if all_levels else {0, 1, 3})
    fd = [f.clone().requires_grad_(True) for f in feats]
    y = U.FPNRoIAlign(7, 7, SCALES)(fd, rois)
    dy = torch.randn(y.shape, generator=g).to(dev)
    y.backward(dy)
    y64, g64 = _ref_grads(lambda *f: G.fpn_roi_align(list(f), rois, 7, 7, SCALES, 2), feats, dy)
    bd = G.fpn_roi_align_bounds(feats, rois, 7, 7, SCALES, 2, dy)
    _check("roi_y", y, y64, bd["y"], slack=bd["y_slack"])
    for l in range(4):
        _check("roi_dfeat", fd[l].grad, g64[l], bd["feat"][l], "P%d" % (l + 2), slack=bd["feat_slack"][l])
        if l not in lv:
            assert not bool(fd[l].grad.any())


def test_fpn_roi_align_rejects_grad_on_bf16(dev):
    import upsnet_b200 as U
    feats = [torch.randn(1, 8, 32 // 2 ** l, 32 // 2 ** l, device=dev).bfloat16().requires_grad_(True) for l in range(4)]
    with pytest.raises(TypeError):
        U.FPNRoIAlign(7, 7, SCALES)(feats, torch.tensor([[0, 0, 0, 50, 50.]], device=dev))


@pytest.mark.parametrize("modulated", [False, True])
def test_deformable_groups_above_one_with_grad_raises(dev, modulated):
    import upsnet_b200 as U
    m = (U.ModDeformConv if modulated else U.DeformConv)(8, 8, 3, padding=1, deformable_groups=2).to(dev)
    x = torch.randn(1, 8, 6, 6, device=dev)
    om = torch.zeros(1, (27 if modulated else 18) * 2, 6, 6, device=dev)
    with pytest.raises(NotImplementedError):
        m(x, om)
    with torch.no_grad():           # the forward-only path keeps deformable groups
        assert m(x, om).shape == (1, 8, 6, 6)


# ------------------------------------------------------------------------------------------------
# a chain of modules against a float64 twin
# ------------------------------------------------------------------------------------------------
def test_chain_every_parameter_gets_the_fp64_gradient(dev):
    """DCN bottleneck (nn.Conv2d offsets + DeformConv, no bias, dilation 2), two DeformConvWithOffset + ReLU, FPNRoIAlign
    on the result and its 2x / 4x / 8x average pools, nn.Linear, scalar loss.  The twin runs the same graph in float64
    from the restatement; its sample positions take the fp32 offsets the device computed.  The check is per tensor,
    relative to the largest gradient element, since the element bounds of grad_oracle do not compose through a chain."""
    import torch.nn.functional as F
    import upsnet_b200 as U
    from upsnet_b200 import operators as ops
    torch.manual_seed(16)
    C, H, W = 16, 32, 40
    off0 = torch.nn.Conv2d(C, 18, 3, padding=2, dilation=2).to(dev)
    off0.weight.data.normal_(0, 0.05)
    dcn0 = U.DeformConv(C, C, 3, padding=2, dilation=2, bias=False).to(dev)
    layers = [U.DeformConvWithOffset(C, C, 3, padding=1).to(dev) for _ in range(2)]
    for l in layers:
        l.conv_offset.weight.data.normal_(0, 0.05); l.conv_offset.bias.data.normal_(0, 0.3)
    fc = torch.nn.Linear(C * 49, 5).to(dev)
    # one or two rois per level on the 128 x 160 image whose P2 is the 32 x 40 map
    rois = torch.tensor([[0, 80 - s / 2 + d, 64 - s / 2 - d, 80 + s / 2 + d - 1, 64 + s / 2 - d - 1]
                         for s, d in ((40, -30), (60, 25), (120, -7), (130, 12), (250, 3), (300, -20), (460, 0))],
                        dtype=torch.float32, device=dev)
    x = torch.randn(1, C, H, W, device=dev, requires_grad=True)

    def run(xv, p, dcn, offs32=None):
        """p: offset conv 0 weight, bias; layers' (offset w, offset b, w, b); fc w, b.  dcn = restatement or None."""
        outs32 = []
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            o = F.conv2d(xv, p[0], p[1], padding=2, dilation=2)
        if dcn is None:
            outs32.append(o.detach())
            h = dcn0(xv, o)
        else:
            h = dcn(xv, o, p[2], None, None, 1, 2, 2, offset32=offs32[0])
        for i in range(2):
            ow, ob, w, b = p[3 + 4 * i:7 + 4 * i]
            h = torch.relu(h)
            if dcn is None:
                with torch.no_grad():
                    outs32.append(ops.conv2d(h, ow, ob, 1, 1, 1, out_format="nchw"))
                h = layers[i](h)
            else:
                h = dcn(h, F.conv2d(h, ow, ob, padding=1), w, b, None, 1, 1, 1, offset32=offs32[1 + i])
        h = torch.relu(h)
        feats = [h] + [F.avg_pool2d(h, 2 ** k) for k in (1, 2, 3)]
        r = (U.FPNRoIAlign(7, 7, SCALES)(feats, rois) if dcn is None else G.fpn_roi_align(feats, rois, 7, 7, SCALES, 2))
        loss = (F.linear(r.reshape(r.shape[0], -1), p[-2], p[-1]) ** 2).sum()
        return loss, outs32

    params = [off0.weight, off0.bias, dcn0.weight]
    for l in layers:
        params += [l.conv_offset.weight, l.conv_offset.bias, l.conv.weight, l.conv.bias]
    params += [fc.weight, fc.bias]
    loss, offs32 = run(x, params, None)
    loss.backward()
    twin = [t.detach().double().requires_grad_(True) for t in [x] + params]
    loss64, _ = run(twin[0], twin[1:], G.deform_conv, offs32)
    loss64.backward()
    assert abs(float(loss) - float(loss64)) <= 1e-5 * abs(float(loss64))
    for i, (p, q) in enumerate(zip([x] + params, twin)):
        assert p.grad is not None, i
        assert bool(q.grad.any()), i
        err = float((p.grad.double() - q.grad).abs().max())
        assert err <= 1e-4 * float(q.grad.abs().max()), (i, err, float(q.grad.abs().max()))


def test_mask_term_is_differentiable(dev):
    """MaskTerm (training twin of the mask paste) back-propagates to the mask logits through the device tensor ops."""
    import upsnet_b200 as U
    masks = torch.randn(3, 1, 28, 28, device=dev, requires_grad=True)
    boxes = torch.tensor([[0, 8, 8, 100, 90], [0, 40, 20, 160, 120], [0, 0, 0, 30, 30]], dtype=torch.float32, device=dev)
    seg = torch.zeros(1, 19, 48, 80, device=dev)
    e = U.MaskTerm(19, box_scale=0.25)(masks, boxes, torch.tensor([1, 2, 3], device=dev), seg)
    e.sum().backward()
    assert masks.grad is not None and float(masks.grad.abs().sum()) > 0
